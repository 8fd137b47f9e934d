// tests/static_timers_host.cpp - TEST INFRASTRUCTURE: the static tier's timers, resume / yield, waits on processes and events, the
// model's events by handle and observers, compiled for the CPU from the SAME source text on both engines - FrontDeskT (model 8) on
// the general engine (cimba_b200/csrc/cmb_device.cuh) and on cmb::StaticSimOf<ModelT, NPROC, NQUEUE, NEVENT>
// (cimba_b200/csrc/cmb_static.cuh), plus a small model of this file's own - and exported as a small C library, so that
// tests/test_static_timers.py can hold them to the reference trial by trial where there is no GPU.  The CUDA vocabulary is mapped
// to C++ as in tests/cmb_engine_host.cpp.  Not a product path: built by the test.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC static_timers_host.cpp -o libstatic_timers_host.so
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

#include "../cimba_b200/models/coverage_models.cuh"

using namespace cimba_b200;

// Customers with patience: twelve of them arrive, each wants 1 or 2 units of a pool of `servers` (2 in the tests) and sets a timer
// before it waits - a customer that wants 2 and finds 1 grabs it and waits for the other, so a timeout during a partial grab rolls
// it back.  A served customer holds, releases, and yields until the dispatcher resumes it (or a timer of its own tells it to go on
// alone).  An end event stops everybody.  The same text compiles in the tier's first form, where every timer sends the trial away.
// Counters: 0 served, 1 timeouts, 2 timeouts that rolled back a partial grab, 3 resumed by the dispatcher, 4 went on alone,
// 5 resumes issued, 6 timers cancelled by handle, 7 sum of the signals that ended the yields.
template <class S>
struct PatienceT {
    typename S::resourcepool_type pool;
    uint64_t counter[8];
    uint32_t yielded;           // bit i: customer i is yielding, waiting for the dispatcher
    double   sum_wait, arr_mean, srv_mean, patience;
    enum : uint32_t { CUSTOMER, DISPATCHER };
    enum : uint32_t { END_EVENT = cmb::ACT_CMB_USER };
    enum : int64_t { SIG_NEXT = 21, SIG_ALONE = 33 };
    static constexpr uint32_t CUSTOMERS = 12u;
    static constexpr bool static_interrupts = true;
    static constexpr bool static_waits = true;
    static CMB_FN constexpr uint32_t static_kind(uint32_t i) { return i < CUSTOMERS ? CUSTOMER : DISPATCHER; }
    template <class F>
    CMB_FN void static_holdables(F &&visit) { visit(pool); }

    // u[0] = the patience timer's handle, u[1] = the units wanted, f[0] = when it arrived
    CMB_FN void customer(S &sim, uint32_t me, int64_t sig)
    {
        PatienceT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(arr_mean);
            sim.proc[me].f[0] = cmb_time();
            sim.proc[me].u[1] = (uint64_t)cmb_random_dice(1, 2);
            sim.proc[me].u[0] = cmb_process_timer_add(cmb_random_exponential(patience), CMB_PROCESS_TIMEOUT);
            CMB_RESOURCEPOOL_ACQUIRE(pool, sim.proc[me].u[1]);
            if (sig == CMB_PROCESS_SUCCESS) {
                if (cmb_process_timer_cancel(sim.proc[me].u[0])) counter[6] += 1u;
                counter[0] += 1u;
                sum_wait = __dadd_rn(sum_wait, __dsub_rn(cmb_time(), sim.proc[me].f[0]));
                CMB_PROCESS_HOLD_EXPONENTIAL(srv_mean);
                CMB_RESOURCEPOOL_RELEASE(pool, sim.proc[me].u[1]);
                yielded |= 1u << me;
                cmb_process_timer_set(cmb_random_exponential(4.0), SIG_ALONE);
                CMB_PROCESS_YIELD();
                yielded &= ~(1u << me);
                counter[sig == SIG_NEXT ? 3 : 4] += 1u;
                counter[7] += (uint64_t)sig;
                cmb_process_timers_clear(me);
            }
            else {
                counter[1] += 1u;
                if (sim.proc[me].fr[1] < sim.proc[me].u[1]) counter[2] += 1u;
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void dispatcher(S &sim, uint32_t me, int64_t sig)
    {
        PatienceT &m = *this;
        CMB_PROCESS_BEGIN
        for (;;) {
            CMB_PROCESS_HOLD_EXPONENTIAL(0.6);
            if (yielded != 0u) {
                uint32_t pick = (uint32_t)cmb_random_dice(0, (long long)CUSTOMERS - 1);
                while (((yielded >> pick) & 1u) == 0u) pick = (pick + 1u) % CUSTOMERS;
                yielded &= ~(1u << pick);
                cmb_process_resume(pick, SIG_NEXT);
                counter[5] += 1u;
            }
        }
        CMB_PROCESS_END
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        for (uint32_t i = 0u; i < 8u; i++) counter[i] = 0u;
        yielded = 0u;
        sum_wait = 0.0;
        arr_mean = in.arr_mean;
        srv_mean = in.srv_mean;
        patience = __dmul_rn(0.5, in.srv_mean);
        cmb_resourcepool_initialize(pool, (uint64_t)in.servers);
        for (uint32_t i = 0u; i <= CUSTOMERS; i++) cmb_process_start(cmb_process_create(i < CUSTOMERS ? CUSTOMER : DISPATCHER, 0, i));
        (void)cmb_event_schedule(END_EVENT, cmb::NIL, 0, (double)in.num_objects, 0);
    }

    CMB_FN void process(S &sim, uint32_t me, uint32_t kind, int64_t sig)
    {
        if (kind == CUSTOMER) customer(sim, me, sig);
        else dispatcher(sim, me, sig);
    }

    CMB_FN void event(S &sim, uint32_t action, uint32_t, int64_t)
    {
        PatienceT &m = *this;
        if (action == END_EVENT) {
            for (uint32_t i = 0u; i <= CUSTOMERS; i++) cmb_process_stop(i, 0);
        }
    }

    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void finish(S &, cmb::TrialOut &out)
    {
        for (uint32_t i = 0u; i < 8u; i++) out.counters[i] = counter[i];
        out.objects = counter[0];
        out.sum_wait = sum_wait;
        out.max_queue = 0u;
    }
};

constexpr int PATIENCE_NPROC = (int)PatienceT<cmb::Sim>::CUSTOMERS + 1;
constexpr int PATIENCE_NEVENT = 16;     // the end event, a timer per customer, the dispatcher's resume, room to spare

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

// S: the tier's sim for the model - cmb::StaticSimOf<...> as the library's route builds it, or a form chosen by hand
template <template <class> class ModelT, class S>
static void run_static(uint64_t seed, const cmb::TrialIn &in, const ZigHot &hot, HostResult &r, uint64_t trace_cap, uint64_t *tk,
                       double *tt)
{
    S sim;
    ModelT<S> m;
    cmb::TrialOut o;
    double win[cmb::STATIC_WINDOW];
    sim.init(seed, &hot, win, 1u, nullptr, 0u);
    cmb::static_run_trial_host(sim, m, in, o, trace_cap, tk, tt);
    copy_out(sim, o, r);
}

constexpr int FD = models::FRONTDESK_SPARE_SLOTS;
using FrontDeskStatic = cmb::StaticSimOf<models::FrontDeskT, 8, 0, FD>;
using FrontDeskShort = cmb::StaticSimOf<models::FrontDeskT, 8, 0, FD - 1>;
using PatienceStatic = cmb::StaticSimOf<PatienceT, PATIENCE_NPROC, 0, PATIENCE_NEVENT>;
using PatienceFirstForm = cmb::StaticSim<PATIENCE_NPROC, 0, PATIENCE_NEVENT, false, false>;
static_assert(FrontDeskStatic::WAITS && PatienceStatic::WAITS && !PatienceFirstForm::INTERRUPTS, "the forms under test");

extern "C" int host_timers_spare_slots(void) { return FD; }

// model = 8 (FrontDeskT) or 200 (PatienceT, this file's model); engine 0 = the general engine (arena_bytes of growth memory), 1 = the
// static tier as the library's route builds it, 2 = model 8 with ONE spare slot too few (a trial that needs it must be flagged),
// 3 = model 200 in the tier's first form (no static_interrupts: every timer must flag the trial).  trace_cap pops of each trial into
// trace_key / trace_time [count][trace_cap].  Returns 0, -1 for another model or engine.
extern "C" int host_timers_run_trials(int model, int engine, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                                      uint64_t num_objects, double arr_mean, double srv_mean, uint64_t arena_bytes,
                                      uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out)
{
    if ((model != 8 && model != 200) || engine < 0 || engine > 3) return -1;
    if ((model == 8 && engine == 3) || (model == 200 && engine == 2)) return -1;
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
        if (model == 8) {
            if (engine == 0)      run_general<models::FrontDeskT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
            else if (engine == 1) run_static<models::FrontDeskT, FrontDeskStatic>(seed, in, hot, r, trace_cap, tk, tt);
            else                  run_static<models::FrontDeskT, FrontDeskShort>(seed, in, hot, r, trace_cap, tk, tt);
        }
        else {
            if (engine == 0)      run_general<PatienceT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
            else if (engine == 1) run_static<PatienceT, PatienceStatic>(seed, in, hot, r, trace_cap, tk, tt);
            else                  run_static<PatienceT, PatienceFirstForm>(seed, in, hot, r, trace_cap, tk, tt);
        }
    }
    return 0;
}
