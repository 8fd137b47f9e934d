// tests/static_preempt_host.cpp - TEST INFRASTRUCTURE: the three models of the static tier's second form (priorities,
// interrupts, pre-emption) compiled for the CPU from the SAME source text on both engines - ToolT (test/test_resource.c, model
// 14), CheeseT (test/test_resourcepool.c, model 18) and Tutorial2T (tutorial/tut_2_1.c, model 21) on the general engine
// (cimba_b200/csrc/cmb_device.cuh) and on cmb::StaticSimOf<ModelT, NPROC, 0, NEVENT> (cimba_b200/csrc/cmb_static.cuh) - and
// exported as a small C library, so that tests/test_static_preempt.py can hold both to the reference trial by trial where there
// is no GPU.  The CUDA vocabulary is mapped to C++ as in tests/cmb_engine_host.cpp.  Not a product path: built by the test.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC static_preempt_host.cpp -o libstatic_preempt_host.so
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

#include "../cimba_b200/models/workshop_model.cuh"
#include "../cimba_b200/models/cheese_model.cuh"
#include "../cimba_b200/models/tutorial2_model.cuh"

using namespace cimba_b200;

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

template <template <class> class ModelT, int NPROC, int NEVENT>
static void run_static(uint64_t seed, const cmb::TrialIn &in, const ZigHot &hot, HostResult &r, uint64_t trace_cap, uint64_t *tk,
                       double *tt)
{
    using S = cmb::StaticSimOf<ModelT, NPROC, 0, NEVENT>;
    static_assert(S::SLOTS == NPROC + NEVENT, "");
    S sim;
    ModelT<S> m;
    cmb::TrialOut o;
    double win[cmb::STATIC_WINDOW], ring[1];
    sim.init(seed, &hot, win, 1u, ring, 0u);
    cmb::static_run_trial_host(sim, m, in, o, trace_cap, tk, tt);
    copy_out(sim, o, r);
}

// model = 14 (ToolT), 18 (CheeseT) or 21 (Tutorial2T); engine 0 = the general engine (arena_bytes of growth memory),
// 1 = the static tier with the spare event slots the library's route gives the model (2, 6, 8), 2 = the static tier with ONE
// spare slot (too few: a trial that needs more must be flagged).  trace_cap pops of each trial into trace_key / trace_time
// [count][trace_cap].  Returns 0, -1 for another model or engine.
extern "C" int host_preempt_run_trials(int model, int engine, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                                       uint64_t num_objects, double arr_mean, double srv_mean, uint64_t arena_bytes,
                                       uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out)
{
    if ((model != 14 && model != 18 && model != 21) || engine < 0 || engine > 2) return -1;
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
            if (model == 14) run_general<models::ToolT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
            else if (model == 18) run_general<models::CheeseT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
            else run_general<models::Tutorial2T>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
        }
        else if (engine == 1) {
            if (model == 14) run_static<models::ToolT, 4, 2>(seed, in, hot, r, trace_cap, tk, tt);
            else if (model == 18) run_static<models::CheeseT, 6, 6>(seed, in, hot, r, trace_cap, tk, tt);
            else run_static<models::Tutorial2T, 8, 8>(seed, in, hot, r, trace_cap, tk, tt);
        }
        else {
            if (model == 14) run_static<models::ToolT, 4, 1>(seed, in, hot, r, trace_cap, tk, tt);
            else if (model == 18) run_static<models::CheeseT, 6, 1>(seed, in, hot, r, trace_cap, tk, tt);
            else run_static<models::Tutorial2T, 8, 1>(seed, in, hot, r, trace_cap, tk, tt);
        }
    }
    return 0;
}
