// tests/static_coverage_host.cpp - TEST INFRASTRUCTURE: the last fixed-process coverage models on the static tier's second form,
// compiled for the CPU from the SAME source text on both engines - PoolFightT (model 4: a pool with mice that change their own
// priority, rats that pre-empt and a cat that interrupts) and WorkshopT<S, PLAIN> (models 5 and 12: a cmb_buffer with partial puts
// and gets, a polite and a pre-empting worker on a cmb_resource, a nuisance interrupting with priorities) on the general engine
// (cimba_b200/csrc/cmb_device.cuh) and on cmb::StaticSimOf<ModelT, NPROC, NQUEUE, NEVENT> (cimba_b200/csrc/cmb_static.cuh) - and
// exported as a small C library, so that tests/test_static_coverage.py can hold them to the reference trial by trial where there
// is no GPU.  The CUDA vocabulary is mapped to C++ as in tests/cmb_engine_host.cpp.  Not a product path: built by the test.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC static_coverage_host.cpp -o libstatic_coverage_host.so
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
#include "../cimba_b200/models/workshop_model.cuh"

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

constexpr int PF = models::POOLFIGHT_SPARE_SLOTS, WS = models::WORKSHOP_SPARE_SLOTS;
using PoolFightStatic = cmb::StaticSimOf<models::PoolFightT, 6, 0, PF>;
using PoolFightOneSlot = cmb::StaticSimOf<models::PoolFightT, 6, 0, 1>;
using BufferStatic = cmb::StaticSimOf<models::WorkshopBufferT, 7, 0, WS>;
using BufferOneSlot = cmb::StaticSimOf<models::WorkshopBufferT, 7, 0, 1>;
using RecordedStatic = cmb::StaticSimOf<models::WorkshopRecordedT, 7, 0, WS>;
using RecordedOneSlot = cmb::StaticSimOf<models::WorkshopRecordedT, 7, 0, 1>;
static_assert(PoolFightStatic::INTERRUPTS && BufferStatic::INTERRUPTS && RecordedStatic::INTERRUPTS, "the second form");

extern "C" int host_coverage_spare_slots(int model) { return model == 4 ? PF : WS; }

// model = 4, 5 or 12; engine 0 = the general engine (arena_bytes of growth memory), 1 = the static tier as the library's route
// builds it, 2 = the static tier with ONE spare event slot (a trial that needs more must be flagged).  trace_cap pops of each trial
// into trace_key / trace_time [count][trace_cap].  Returns 0, -1 for another model or engine.
extern "C" int host_coverage_run_trials(int model, int engine, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                                        uint64_t num_objects, double arr_mean, double srv_mean, uint64_t arena_bytes,
                                        uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out)
{
    if ((model != 4 && model != 5 && model != 12) || engine < 0 || engine > 2) return -1;
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
        if (model == 4) {
            if (engine == 0)      run_general<models::PoolFightT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
            else if (engine == 1) run_static<models::PoolFightT, PoolFightStatic>(seed, in, hot, r, trace_cap, tk, tt);
            else                  run_static<models::PoolFightT, PoolFightOneSlot>(seed, in, hot, r, trace_cap, tk, tt);
        }
        else if (model == 5) {
            if (engine == 0)      run_general<models::WorkshopBufferT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
            else if (engine == 1) run_static<models::WorkshopBufferT, BufferStatic>(seed, in, hot, r, trace_cap, tk, tt);
            else                  run_static<models::WorkshopBufferT, BufferOneSlot>(seed, in, hot, r, trace_cap, tk, tt);
        }
        else {
            if (engine == 0)      run_general<models::WorkshopRecordedT>(seed, in, hot, mem, arena_bytes, r, trace_cap, tk, tt);
            else if (engine == 1) run_static<models::WorkshopRecordedT, RecordedStatic>(seed, in, hot, r, trace_cap, tk, tt);
            else                  run_static<models::WorkshopRecordedT, RecordedOneSlot>(seed, in, hot, r, trace_cap, tk, tt);
        }
    }
    return 0;
}
