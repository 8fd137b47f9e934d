// summary.cuh - cmb_datasummary arithmetic (host + device) and the on-device
// reduction of per-trial results.
//
// Reference: src/cmb_datasummary.c:144-166 (add: Pebay's single-sample update in
// Meng's evaluation order) and :93-131 (merge: Pebay's pairwise formula).  The
// benchmark folds the per-trial averages with a serial host loop
// (benchmark/MM1_multi.c:143-148); here each GPU folds its shard with a fixed,
// deterministic tree of the same two operations, and ranks are merged in rank
// order after an all-gather (SURVEY.md section 8e).  A merged tree differs from
// the serial fold by rounding only (<< 1e-9 relative).
//
// Compiled with -fmad=false: the expressions below keep the reference's
// operation order and must not be contracted.
#pragma once

#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#ifndef CMB_HOST_BUILD     // tests/cmb_engine_host.cpp compiles this text for the CPU
#include <cuda_runtime.h>
#endif

namespace cimba_b200 {

struct SummaryAcc {
    uint64_t count;
    double min, max, m1, m2, m3, m4;
};

__host__ __device__ inline SummaryAcc summary_empty()
{
    return SummaryAcc{0u, DBL_MAX, -DBL_MAX, 0.0, 0.0, 0.0, 0.0};
}

// cmb_datasummary_add, src/cmb_datasummary.c:144-166
__host__ __device__ inline void summary_add(SummaryAcc &s, double y)
{
    s.max = (y > s.max) ? y : s.max;
    s.min = (y < s.min) ? y : s.min;

    const double d = y - s.m1;
    const double d_2 = d * d;
    const double d_3 = d * d_2;
    const double n = (double)(++s.count);
    const double d_n = d / n;
    const double d_n_2 = d_n * d_n;
    const double d_n_3 = d_n_2 * d_n;

    s.m1 += d_n;
    s.m2 += d * (d - d_n);
    s.m3 += d * (d_2 - d_n_2) - 3.0 * d_n * s.m2;
    s.m4 += d * (d_3 - d_n_3) - 6.0 * d_n_2 * s.m2 - 4.0 * d_n * s.m3;
}

// cmb_datasummary_merge, src/cmb_datasummary.c:93-131.  An empty side is passed
// through unchanged (the reference formula would divide 0/0 for two empties).
__host__ __device__ inline SummaryAcc summary_merge(const SummaryAcc &a, const SummaryAcc &b)
{
    if (b.count == 0u) {
        return a;
    }
    if (a.count == 0u) {
        return b;
    }
    SummaryAcc c;
    c.count = a.count + b.count;
    c.min = (a.min < b.min) ? a.min : b.min;
    c.max = (a.max > b.max) ? a.max : b.max;

    const double n1 = (double)a.count;
    const double n2 = (double)b.count;
    const double n = (double)c.count;
    const double d21 = b.m1 - a.m1;
    const double d21_n = d21 / n;
    const double d21_n_2 = d21_n * d21_n;
    const double d21_n_3 = d21_n * d21_n_2;

    c.m1 = a.m1 + n2 * d21_n;
    c.m2 = a.m2 + b.m2 + n1 * n2 * d21 * d21_n;
    c.m3 = a.m3 + b.m3
         + n1 * n2 * (n1 - n2) * d21 * d21_n_2
         + 3.0 * (n1 * b.m2 - n2 * a.m2) * d21_n;
    c.m4 = a.m4 + b.m4
         + n1 * n2 * (n1 * n1 - n1 * n2 + n2 * n2) * d21 * d21_n_3
         + 6.0 * (n1 * n1 * b.m2 + n2 * n2 * a.m2) * d21_n_2
         + 4.0 * (n1 * b.m3 - n2 * a.m3) * d21_n;
    return c;
}

// ---- cmb_wtdsummary: the same moments with arbitrary non-negative weights
struct WtdAcc {
    uint64_t count;
    double min, max, m1, m2, m3, m4, wsum;
};

__host__ __device__ inline WtdAcc wtd_empty()
{
    return WtdAcc{0u, DBL_MAX, -DBL_MAX, 0.0, 0.0, 0.0, 0.0, 0.0};
}

// cmb_wtdsummary_add, src/cmb_wtdsummary.c:82-137
__host__ __device__ inline void wtd_add(WtdAcc &s, double x, double w)
{
    if (w == 0.0) {
        return;
    }
    if (s.count == 0u) {
        s.count = 1u;
        s.max = x;
        s.min = x;
        s.m1 = x;
        s.m2 = s.m3 = s.m4 = 0.0;
        s.wsum = w;
        return;
    }
    s.max = (x > s.max) ? x : s.max;
    s.min = (x < s.min) ? x : s.min;
    s.count++;

    const double w1 = s.wsum;
    const double w2 = w;
    const double ws = w1 + w2;
    const double d21 = x - s.m1;
    const double d21_w = d21 / ws;
    const double d21_w_2 = d21_w * d21_w;
    const double d21_w_3 = d21_w * d21_w_2;

    const double m1 = s.m1 + w2 * d21_w;
    const double m2 = s.m2 + w1 * w2 * d21 * d21_w;
    const double m3 = s.m3
                    + w1 * w2 * (w1 - w2) * d21 * d21_w_2
                    - 3.0 * w2 * s.m2 * d21_w;
    const double m4 = s.m4
                    + w1 * w2 * (w1 * w1 - w1 * w2 + w2 * w2) * d21 * d21_w_3
                    + 6.0 * w2 * w2 * s.m2 * d21_w_2
                    - 4.0 * w2 * s.m3 * d21_w;
    s.m1 = m1;
    s.m2 = m2;
    s.m3 = m3;
    s.m4 = m4;
    s.wsum = ws;
}

// cmb_wtdsummary_merge, src/cmb_wtdsummary.c:152-194.  An empty side is passed through
// unchanged (two empties would divide 0/0 in the reference formula).
__host__ __device__ inline WtdAcc wtd_merge(const WtdAcc &a, const WtdAcc &b)
{
    if (b.count == 0u) {
        return a;
    }
    if (a.count == 0u) {
        return b;
    }
    WtdAcc c;
    c.count = a.count + b.count;
    c.min = (a.min < b.min) ? a.min : b.min;
    c.max = (a.max > b.max) ? a.max : b.max;

    const double w1 = a.wsum;
    const double w2 = b.wsum;
    const double ws = w1 + w2;
    const double d21 = b.m1 - a.m1;
    const double d21_w = d21 / ws;
    const double d21_w_2 = d21_w * d21_w;
    const double d21_w_3 = d21_w * d21_w_2;

    c.wsum = ws;
    c.m1 = a.m1 + w2 * d21_w;
    c.m2 = a.m2 + b.m2
         + w1 * w2 * d21 * d21_w;
    c.m3 = a.m3 + b.m3
         + w1 * w2 * (w1 - w2) * d21 * d21_w_2
         + 3.0 * (w1 * b.m2 - w2 * a.m2) * d21_w;
    c.m4 = a.m4 + b.m4
         + w1 * w2 * (w1 * w1 - w1 * w2 + w2 * w2) * d21 * d21_w_3
         + 6.0 * (w1 * w1 * b.m2 + w2 * w2 * a.m2) * d21_w_2
         + 4.0 * (w1 * b.m3 - w2 * a.m3) * d21_w;
    return c;
}

// cmb_datasummary_add / _merge and cmb_wtdsummary_add / _merge as the reference calls them: through pointers, returning the count
__host__ __device__ inline uint64_t summary_add_ptr(SummaryAcc *s, double y)
{
    summary_add(*s, y);
    return s->count;
}

__host__ __device__ inline uint64_t summary_merge_ptr(SummaryAcc *tgt, const SummaryAcc *a, const SummaryAcc *b)
{
    *tgt = summary_merge(*a, *b);
    return tgt->count;
}

__host__ __device__ inline uint64_t wtd_add_ptr(WtdAcc *s, double x, double w)
{
    wtd_add(*s, x, w);
    return s->count;
}

__host__ __device__ inline uint64_t wtd_merge_ptr(WtdAcc *tgt, const WtdAcc *a, const WtdAcc *b)
{
    *tgt = wtd_merge(*a, *b);
    return tgt->count;
}

// ---- the reference's statistics of a summary (include/cmb_datasummary.h, src/cmb_datasummary.c:214-249); cmb_wtdsummary's
// delegate to the same moments (include/cmb_wtdsummary.h:192-197).  A is SummaryAcc, WtdAcc or the C ABI's
// cimba_b200_datasummary: the host's cimba_b200_datasummary_* (capi.cu) and model code (cmb_datasummary_* in cmb_device.cuh)
// both use these.
template <class A>
__host__ __device__ inline double summary_variance(const A &s)      // include/cmb_datasummary.h:197-210 (sample variance)
{
    return (s.count > 1u) ? s.m2 / (double)(s.count - 1u) : 0.0;
}

template <class A>
__host__ __device__ inline double summary_stddev(const A &s)
{
    return sqrt(summary_variance(s));
}

template <class A>
__host__ __device__ inline double summary_skewness(const A &s)      // :214-230: population estimate, then the finite-sample correction
{
    if (s.count <= 2u) return 0.0;
    const double n = (double)s.count;
    const double g = sqrt(n) * s.m3 / pow(s.m2, 1.5);
    return sqrt(n * (n - 1.0)) * g / (n - 2.0);
}

template <class A>
__host__ __device__ inline double summary_kurtosis(const A &s)      // :233-249: sample excess kurtosis
{
    if (s.count <= 3u) return 0.0;
    const double n = (double)s.count;
    const double g = n * s.m4 / (s.m2 * s.m2) - 3.0;
    return (n - 1.0) / ((n - 2.0) * (n - 3.0)) * ((n + 1.0) * g + 6.0);
}

// A summary as one trial's 8-word row of counters: {count (u64), min, max, m1, m2, m3, m4, wsum (f64 bit patterns)} - what
// cimba_b200_merge_weighted_rows reads.  A cmb_datasummary's row carries wsum = count: the weighted merge with weights equal to
// the counts is the unweighted merge (src/cmb_wtdsummary.c:152-194 with w = n is src/cmb_datasummary.c:93-131, term for term).
__host__ __device__ inline uint64_t summary_bits(double d)
{
#ifdef __CUDA_ARCH__
    return (uint64_t)__double_as_longlong(d);
#else
    uint64_t u;
    memcpy(&u, &d, sizeof u);
    return u;
#endif
}

__host__ __device__ inline void wtd_store_row(const WtdAcc &a, uint64_t *row)
{
    row[0] = a.count;
    row[1] = summary_bits(a.min);
    row[2] = summary_bits(a.max);
    row[3] = summary_bits(a.m1);
    row[4] = summary_bits(a.m2);
    row[5] = summary_bits(a.m3);
    row[6] = summary_bits(a.m4);
    row[7] = summary_bits(a.wsum);
}

__host__ __device__ inline void summary_store_row(const WtdAcc &a, uint64_t *row)
{
    wtd_store_row(a, row);
}

__host__ __device__ inline void summary_store_row(const SummaryAcc &a, uint64_t *row)
{
    wtd_store_row(WtdAcc{a.count, a.min, a.max, a.m1, a.m2, a.m3, a.m4, (double)a.count}, row);
}

// A fused cmb_timeseries (src/cmb_timeseries.c:106-188): a new sample fixes the duration of
// the previous one, and that (x, duration) pair is all cmb_timeseries_summarize feeds to
// cmb_wtdsummary_add - so the history itself is never stored.
struct TimeWeighted {
    WtdAcc   acc;
    double   x, t;
    uint32_t n;

    __host__ __device__ inline void start()
    {
        acc = wtd_empty();
        x = t = 0.0;
        n = 0u;
    }
    __host__ __device__ inline void sample(double value, double now)    // cmb_timeseries_add
    {
        if (n != 0u) {
            wtd_add(acc, x, now - t);
        }
        x = value;
        t = now;
        n = 1u;
    }
};

// the same, out of line, for code that samples in many places (general-path kernels)
__device__ __noinline__ void time_weighted_sample(TimeWeighted &h, double value, double now)
{
    h.sample(value, now);
}

#ifndef CMB_HOST_BUILD     // the reduction kernels below are device-only
constexpr int SUMMARY_BLOCK = 256;

// One CTA: thread t adds trials t, t+256, ... (coalesced reads), then a fixed
// halving tree of merges in shared memory.  out = {count,min,max,m1,m2,m3,m4,0}.
__global__ void __launch_bounds__(SUMMARY_BLOCK)
summarize_kernel(const double *__restrict__ sum_wait, const uint64_t *__restrict__ objects,
                 uint64_t n, double *__restrict__ out)
{
    __shared__ SummaryAcc part[SUMMARY_BLOCK];
    SummaryAcc acc = summary_empty();
    for (uint64_t i = threadIdx.x; i < n; i += SUMMARY_BLOCK) {
        // avg_tsys = sum_wait / (double)obj_cnt, benchmark/MM1_multi.c:146
        summary_add(acc, sum_wait[i] / (double)objects[i]);
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    for (int s = SUMMARY_BLOCK / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            part[threadIdx.x] = summary_merge(part[threadIdx.x], part[threadIdx.x + s]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const SummaryAcc r = part[0];
        out[0] = (double)r.count;
        out[1] = r.min;
        out[2] = r.max;
        out[3] = r.m1;
        out[4] = r.m2;
        out[5] = r.m3;
        out[6] = r.m4;
        out[7] = 0.0;
    }
}

// The weighted counterparts.  rows[i] = one trial's cmb_wtdsummary as the engine writes it
// into counters[i][0..7]: {count (u64), min, max, m1, m2, m3, m4, wsum (f64 bit patterns)}.
__device__ inline WtdAcc wtd_load_row(const uint64_t *row)
{
    WtdAcc a;
    a.count = row[0];
    a.min = __longlong_as_double((long long)row[1]);
    a.max = __longlong_as_double((long long)row[2]);
    a.m1 = __longlong_as_double((long long)row[3]);
    a.m2 = __longlong_as_double((long long)row[4]);
    a.m3 = __longlong_as_double((long long)row[5]);
    a.m4 = __longlong_as_double((long long)row[6]);
    a.wsum = __longlong_as_double((long long)row[7]);
    return a;
}

__device__ inline void wtd_block_reduce(WtdAcc acc, uint64_t *out_row)
{
    __shared__ WtdAcc part[SUMMARY_BLOCK];
    part[threadIdx.x] = acc;
    __syncthreads();
    for (int s = SUMMARY_BLOCK / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            part[threadIdx.x] = wtd_merge(part[threadIdx.x], part[threadIdx.x + s]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        wtd_store_row(part[0], out_row);
    }
}

// cmb_wtdsummary_add over (x[i], w[i]): thread t adds samples t, t+256, ..., then the merge tree.
__global__ void __launch_bounds__(SUMMARY_BLOCK)
summarize_weighted_kernel(const double *__restrict__ x, const double *__restrict__ w,
                          uint64_t n, uint64_t *__restrict__ out_row)
{
    WtdAcc acc = wtd_empty();
    for (uint64_t i = threadIdx.x; i < n; i += SUMMARY_BLOCK) {
        wtd_add(acc, x[i], w[i]);
    }
    wtd_block_reduce(acc, out_row);
}

// cmb_wtdsummary_merge over per-trial summaries (rows of 8 words): thread t folds rows
// t, t+256, ... in index order, then the merge tree.
__global__ void __launch_bounds__(SUMMARY_BLOCK)
merge_weighted_rows_kernel(const uint64_t *__restrict__ rows, uint64_t n, uint64_t *__restrict__ out_row)
{
    WtdAcc acc = wtd_empty();
    for (uint64_t i = threadIdx.x; i < n; i += SUMMARY_BLOCK) {
        acc = wtd_merge(acc, wtd_load_row(rows + i * 8u));
    }
    wtd_block_reduce(acc, out_row);
}

#endif  // CMB_HOST_BUILD

}  // namespace cimba_b200
