// tests/cmb_engine_host.cpp - TEST INFRASTRUCTURE: the general engine (cimba_b200/csrc/cmb_device.cuh) and the models
// written against its authoring surface (cimba_b200/models/*.cuh), compiled for the CPU from the SAME source text and
// exported as a small C library, so that tests/test_cmb_engine.py can hold them to the reference build
// (oracle/_ref/librefdrv.so) trial by trial where there is no GPU.  One trial per call frame, no warp-level anything:
// the engine is lane-per-trial, so the host build is the device code with the CUDA vocabulary mapped to C++.
// Not a product path: built by the test, under tests/.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC cmb_engine_host.cpp -o libcmb_engine_host.so
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

#include "../cimba_b200/models/mm1_model.cuh"
#include "../cimba_b200/models/mm1_recorded_model.cuh"
#include "../cimba_b200/models/tutorial1_model.cuh"
#include "../cimba_b200/models/park_model.cuh"
#include "../cimba_b200/models/tutorial2_model.cuh"
#include "../cimba_b200/models/mmc_model.cuh"
#include "../cimba_b200/models/renege_model.cuh"
#include "../cimba_b200/models/gg1_model.cuh"
#include "../cimba_b200/models/hold_general_model.cuh"
#include "../cimba_b200/models/cheese_model.cuh"
#include "../cimba_b200/models/harbor_general_model.cuh"
#include "../cimba_b200/models/guarded_model.cuh"
#include "../cimba_b200/models/workshop_model.cuh"
#include "../cimba_b200/models/coverage_models.cuh"
#include "../examples/tandem_model.cuh"

using namespace cimba_b200;

struct HostResult {
    uint64_t events, objects;
    double   t_end, sum_wait;
    uint64_t max_fel, max_queue;
    uint64_t counter[8];
    uint32_t status, pad;
};

template <class Model>
static void run_model(uint64_t seed, const cmb::TrialIn &in, cmb::Arena &arena, const ZigHot &hot, HostResult &r,
                      uint64_t trace_cap, uint64_t *trace_key, double *trace_time)
{
    cmb::Sim sim;
    Model m;
    cmb::TrialOut out;
    sim.init(seed, &hot, arena);
    if (trace_cap) cmb::run_one_trial<Model, true>(sim, m, in, out, trace_cap, trace_key, trace_time);
    else           cmb::run_one_trial<Model, false>(sim, m, in, out, 0u, nullptr, nullptr);
    r.events = sim.pops;
    r.objects = out.objects;
    r.t_end = sim.now;
    r.sum_wait = out.sum_wait;
    r.max_fel = sim.fel.cap();
    r.max_queue = out.max_queue;
    std::memcpy(r.counter, out.counters, sizeof(r.counter));
    r.status = sim.status;
    r.pad = 0u;
}

// the static tier (csrc/cmb_static.cuh): the same model template on cmb::StaticSim; spill_cap entries of HBM-ring stand-in per queue
template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT = 0>
static void run_static(uint64_t seed, const cmb::TrialIn &in, const ZigHot &hot, HostResult &r, uint32_t spill_cap,
                       uint64_t trace_cap, uint64_t *trace_key, double *trace_time)
{
    using S = cmb::StaticSim<NPROC, NQUEUE, NEVENT>;
    S sim;
    ModelT<S> m;
    cmb::TrialOut out;
    std::vector<double> win((size_t)(NQUEUE + 1) * cmb::STATIC_WINDOW), ring((size_t)(NQUEUE + 1) * (spill_cap ? spill_cap : 1u));
    sim.init(seed, &hot, win.data(), 1u, ring.data(), spill_cap);
    cmb::static_run_trial_host(sim, m, in, out, trace_cap, trace_key, trace_time);
    r.events = sim.pops;
    r.objects = out.objects;
    r.t_end = sim.now;
    r.sum_wait = out.sum_wait;
    r.max_fel = NPROC;
    r.max_queue = out.max_queue;
    std::memcpy(r.counter, out.counters, sizeof(r.counter));
    r.status = sim.status;
    r.pad = 0u;
}

// model + 100 = the same model on the static tier (arena_bytes then = entries of the HBM-ring stand-in per queue).
// model: 0 = MM1, 1 = GG1, 2 = MMC, 3 / 11 / 13 = the guarded queue tests, 5 / 12 = buffer + resource, 14 = test_resource.c, 7 = HOLD, 10 = HARBOR, 16 = RENEGE (the CIMBA_B200_MODEL_* numbers), 17 = examples/tandem_model.cuh, 18 = CHEESE (test/test_resourcepool.c).  arena_bytes of growth memory per call.
// arena_used (may be NULL): per trial, the arena cursor when the trial ended - the bytes its containers asked for, granted
// or not.  Allocation order is fixed by the seed, so a trial runs unflagged exactly when arena_bytes >= that figure.
static int run_trials(int model, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                      uint64_t num_objects, double arr_mean, double srv_mean,
                      const double *params, uint32_t num_params, uint64_t arena_bytes,
                      uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out, uint64_t *arena_used)
{
    static ZigHot hot;
    for (int i = 0; i < 256; i++) {
        hot.exp_x[i] = zig::zig_exp_x[i];
        hot.nor_x[i] = zig::zig_nor_x[i];
    }
    std::vector<unsigned char> mem((model >= 100 ? 0u : arena_bytes) + 256);
    for (uint64_t i = 0; i < count; i++) {
        unsigned long long cursor = 0;
        cmb::Arena arena{mem.data(), &cursor, arena_bytes};
        cmb::TrialIn in{};
        in.arr_mean = arr_mean;
        in.srv_mean = srv_mean;
        in.num_objects = num_objects;
        in.servers = servers;
        in.num_params = num_params;
        for (uint32_t k = 0; k < num_params && k < 16u; k++) in.params[k] = params[k];
        in.trial = first + i;
        const uint64_t seed = fmix64(master_seed, first + i);
        uint64_t *tk = trace_cap ? trace_key + i * trace_cap : nullptr;
        double *tt = trace_cap ? trace_time + i * trace_cap : nullptr;
        switch (model) {
        case 0:  run_model<models::MM1>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 21: run_model<models::Tutorial2>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 20: run_model<models::Park>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 19: run_model<models::Tutorial1>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 9:  run_model<models::MM1Recorded>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 119: run_static<models::Tutorial1T, 2, 0, 3>(seed, in, hot, out[i], (uint32_t)arena_bytes, trace_cap, tk, tt); break;
        case 109: run_static<models::MM1RecordedT, 2, 1>(seed, in, hot, out[i], (uint32_t)arena_bytes, trace_cap, tk, tt); break;
        case 100: run_static<models::MM1T, 2, 1>(seed, in, hot, out[i], (uint32_t)arena_bytes, trace_cap, tk, tt); break;
        case 101: run_static<models::GG1T, 2, 1>(seed, in, hot, out[i], (uint32_t)arena_bytes, trace_cap, tk, tt); break;
        case 117: run_static<tandem_example::TandemT, 3, 2>(seed, in, hot, out[i], (uint32_t)arena_bytes, trace_cap, tk, tt); break;
        case 1:  run_model<models::GG1>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 7:  run_model<models::HoldGeneral>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 10: run_model<models::HarborGeneral>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 3:  run_model<models::Guarded<false, false>>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 11: run_model<models::Guarded<false, true>>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 13: run_model<models::Guarded<true, true>>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 5:  run_model<models::Workshop<false>>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 12: run_model<models::Workshop<true>>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 14: run_model<models::Tool>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 4:  run_model<models::PoolFight>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 6:  run_model<models::QueueAndTide>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 8:  run_model<models::FrontDesk>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 18: run_model<models::Cheese>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 17: run_model<tandem_example::Tandem>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 2:  run_model<models::MMC>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        case 16: run_model<models::Renege>(seed, in, arena, hot, out[i], trace_cap, tk, tt); break;
        default: return -1;
        }
        if (arena_used) arena_used[i] = cursor;
    }
    return 0;
}

extern "C" int host_cmb_run_trials(int model, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                                   uint64_t num_objects, double arr_mean, double srv_mean,
                                   const double *params, uint32_t num_params, uint64_t arena_bytes,
                                   uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out)
{
    return run_trials(model, servers, master_seed, first, count, num_objects, arr_mean, srv_mean, params, num_params, arena_bytes,
                      trace_cap, trace_key, trace_time, out, nullptr);
}

// host_cmb_run_trials + each trial's arena cursor (tests/test_growth_arena.py)
extern "C" int host_cmb_run_trials_used(int model, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                                        uint64_t num_objects, double arr_mean, double srv_mean,
                                        const double *params, uint32_t num_params, uint64_t arena_bytes,
                                        uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out,
                                        uint64_t *arena_used)
{
    return run_trials(model, servers, master_seed, first, count, num_objects, arr_mean, srv_mean, params, num_params, arena_bytes,
                      trace_cap, trace_key, trace_time, out, arena_used);
}
