// tests/static_queues_host.cpp - TEST INFRASTRUCTURE: the models of the static tier that use cmb_priorityqueue and cmb_condition,
// compiled for the CPU from the SAME source text on both engines - GuardedT (test/test_objectqueue.c and test/test_priorityqueue.c,
// models 3, 11 and 13) and QueueAndTideT (model 6) on the general engine (cimba_b200/csrc/cmb_device.cuh) and on
// cmb::StaticSimOf<ModelT, NPROC, NQUEUE, NEVENT> (cimba_b200/csrc/cmb_static.cuh), plus a small model of this file's own in the
// tier's first form (no static_interrupts) - and exported as a small C library, so that tests/test_static_queues.py can hold them
// to the reference trial by trial where there is no GPU.  The CUDA vocabulary is mapped to C++ as in tests/cmb_engine_host.cpp.
// Not a product path: built by the test.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC static_queues_host.cpp -o libstatic_queues_host.so
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

#include "../cimba_b200/models/guarded_model.cuh"
#include "../cimba_b200/models/coverage_models.cuh"

using namespace cimba_b200;

// The tier's first form (no static_interrupts, every process at priority 0): a two-class priority M/M/1 - arrivals put their
// time stamp into a priority queue at class 0 or 1, one server takes the highest class first - and an observer that waits on a
// condition until the queue is LONG, counting each time it gets through.  The arrivals signal the condition after each put;
// after num_objects arrivals the arrival process exits and the event list runs dry.
template <class S>
struct TwoClassT {
    typename S::priorityqueue_type line;
    typename S::condition_type     long_line;
    uint64_t counter[8];
    uint64_t arrivals;
    double   sum_wait, arr_mean, srv_mean;
    enum : uint32_t { ARRIVAL, SERVER, OBSERVER };
    enum : uint32_t { LONG = 7u };
    static constexpr uint64_t LONG_AT = 3u;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i; }

    // u[0] = the object in hand, u[1] = the handle of the last put
    CMB_FN void arrival(S &sim, uint32_t me, int64_t sig)
    {
        TwoClassT &m = *this;
        CMB_PROCESS_BEGIN
        while (arrivals < num_objects) {
            CMB_PROCESS_HOLD_EXPONENTIAL(arr_mean);
            arrivals++;
            sim.proc[me].u[0] = (uint64_t)__double_as_longlong(cmb_time());
            sim.proc[me].f[0] = (double)cmb_random_dice(0, 1);
            CMB_PRIORITYQUEUE_PUT(line, sim.proc[me].u[0], (int64_t)sim.proc[me].f[0], &sim.proc[me].u[1]);
            counter[sim.proc[me].f[0] > 0.5 ? 1 : 0] += 1u;
            counter[7] = sim.proc[me].u[1];
            if (cmb_priorityqueue_position(line, sim.proc[me].u[1]) == 1u) counter[6] += 1u;
            counter[4] += cmb_condition_signal(long_line);
        }
        CMB_PROCESS_END
    }

    CMB_FN void server(S &sim, uint32_t me, int64_t sig)
    {
        TwoClassT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PRIORITYQUEUE_GET(line, sim.proc[me].u[0]);
            sum_wait = __dadd_rn(sum_wait, __dsub_rn(cmb_time(), __longlong_as_double((long long)sim.proc[me].u[0])));
            CMB_PROCESS_HOLD_EXPONENTIAL(srv_mean);
            counter[2] += 1u;
        }
        CMB_PROCESS_END
    }

    CMB_FN void observer(S &sim, uint32_t me, int64_t sig)
    {
        TwoClassT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            while (cmb_priorityqueue_length(line) < LONG_AT) CMB_CONDITION_WAIT(long_line, LONG, 0);
            counter[5] += 1u;
            CMB_PROCESS_HOLD_EXPONENTIAL(2.0);
        }
        CMB_PROCESS_END
    }

    uint64_t num_objects;

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        for (uint32_t i = 0u; i < 8u; i++) counter[i] = 0u;
        arrivals = 0u;
        sum_wait = 0.0;
        arr_mean = in.arr_mean;
        srv_mean = in.srv_mean;
        num_objects = in.num_objects;
        cmb_priorityqueue_initialize(line, (uint64_t)in.servers);
        cmb_condition_initialize(long_line);
        for (uint32_t i = 0u; i < 3u; i++) cmb_process_start(cmb_process_create(i, 0, i));
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == ARRIVAL) arrival(sim, me, sig);
        else if (kind == SERVER) server(sim, me, sig);
        else observer(sim, me, sig);
    }

    CMB_FN void event(S &, uint32_t, uint32_t, int64_t) {}
    CMB_FN bool demand(S &, uint32_t id, uint32_t, int32_t) { return id == LONG && cmb::priorityqueue_length(line) >= LONG_AT; }

    CMB_FN void finish(S &, cmb::TrialOut &out)
    {
        counter[3] = cmb::priorityqueue_length(line);
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.objects = counter[2];
        out.sum_wait = sum_wait;
        out.max_queue = 0u;
    }
};

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

template <template <class> class ModelT>
static void run_general(uint64_t seed, const cmb::TrialIn &in, const ZigHot &hot, std::vector<unsigned char> &mem, uint64_t arena_bytes,
                        HostResult &r, uint64_t trace_cap, uint64_t *tk, double *tt)
{
    unsigned long long cursor = 0;
    cmb::Arena arena{mem.data(), &cursor, arena_bytes};
    cmb::Sim sim;
    ModelT<cmb::Sim> m;
    cmb::TrialOut o;
    sim.init(seed, &hot, arena);
    if (trace_cap) cmb::run_one_trial<ModelT<cmb::Sim>, true>(sim, m, in, o, trace_cap, tk, tt);
    else           cmb::run_one_trial<ModelT<cmb::Sim>, false>(sim, m, in, o, 0u, nullptr, nullptr);
    copy_out(sim, o, r);
}

// the queue window only, no HBM ring: as the library's route launches these models
template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT>
static void run_static(uint64_t seed, const cmb::TrialIn &in, const ZigHot &hot, HostResult &r, uint64_t trace_cap, uint64_t *tk,
                       double *tt)
{
    using S = cmb::StaticSimOf<ModelT, NPROC, NQUEUE, NEVENT>;
    static_assert(S::SLOTS == NPROC + NEVENT, "");
    S sim;
    ModelT<S> m;
    cmb::TrialOut o;
    double win[(NQUEUE > 0 ? NQUEUE : 1) * cmb::STATIC_WINDOW];
    sim.init(seed, &hot, win, 1u, nullptr, 0u);
    cmb::static_run_trial_host(sim, m, in, o, trace_cap, tk, tt);
    copy_out(sim, o, r);
}

template <class S> using Guarded3 = models::GuardedQueueT<S>;
template <class S> using Guarded11 = models::GuardedRecordedQueueT<S>;
template <class S> using Guarded13 = models::GuardedPriorityQueueT<S>;

// model = 3, 11, 13 (GuardedT), 6 (QueueAndTideT) or 100 (TwoClassT, this file's first-form model); engine 0 = the general
// engine (arena_bytes of growth memory), 1 = the static tier with the spare event slots the library's route gives the model
// (2; none for model 100), 2 = the static tier with ONE spare slot (one too few: a trial that needs more must be flagged).
// trace_cap pops of each trial into trace_key / trace_time [count][trace_cap].  Returns 0, -1 for another model or engine.
extern "C" int host_queues_run_trials(int model, int engine, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                                      uint64_t num_objects, double arr_mean, double srv_mean, uint64_t arena_bytes,
                                      uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out)
{
    if ((model != 3 && model != 6 && model != 11 && model != 13 && model != 100) || engine < 0 || engine > 2) return -1;
    if (model == 100 && engine == 2) return -1;
    static ZigHot hot;
    for (int i = 0; i < 256; i++) {
        hot.exp_x[i] = zig::zig_exp_x[i];
        hot.nor_x[i] = zig::zig_nor_x[i];
    }
    std::vector<unsigned char> mem((engine == 0 ? arena_bytes : 0u) + 256);
    for (uint64_t i = 0; i < count; i++) {
        cmb::TrialIn in{};
        in.arr_mean = arr_mean;
        in.srv_mean = srv_mean;
        in.num_objects = num_objects;
        in.servers = servers;
        in.trial = first + i;
        const uint64_t seed = fmix64(master_seed, first + i);
        uint64_t *tk = trace_cap ? trace_key + i * trace_cap : nullptr;
        double *tt = trace_cap ? trace_time + i * trace_cap : nullptr;
        HostResult &r = out[i];
        if (engine == 0) {
            switch (model) {
            case 3:  run_general<Guarded3>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt); break;
            case 11: run_general<Guarded11>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt); break;
            case 13: run_general<Guarded13>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt); break;
            case 6:  run_general<models::QueueAndTideT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt); break;
            default: run_general<TwoClassT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt); break;
            }
        }
        else if (engine == 1) {
            switch (model) {
            case 3:  run_static<Guarded3, 7, 1, 2>(seed, in, hot, r, trace_cap, tk, tt); break;
            case 11: run_static<Guarded11, 7, 1, 2>(seed, in, hot, r, trace_cap, tk, tt); break;
            case 13: run_static<Guarded13, 7, 0, 2>(seed, in, hot, r, trace_cap, tk, tt); break;
            case 6:  run_static<models::QueueAndTideT, 8, 0, 2>(seed, in, hot, r, trace_cap, tk, tt); break;
            default: run_static<TwoClassT, 3, 0, 0>(seed, in, hot, r, trace_cap, tk, tt); break;
            }
        }
        else {
            switch (model) {
            case 3:  run_static<Guarded3, 7, 1, 1>(seed, in, hot, r, trace_cap, tk, tt); break;
            case 11: run_static<Guarded11, 7, 1, 1>(seed, in, hot, r, trace_cap, tk, tt); break;
            case 13: run_static<Guarded13, 7, 0, 1>(seed, in, hot, r, trace_cap, tk, tt); break;
            default: run_static<models::QueueAndTideT, 8, 0, 1>(seed, in, hot, r, trace_cap, tk, tt); break;
            }
        }
    }
    return 0;
}
