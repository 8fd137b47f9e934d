// tests/static_resources_host.cpp - TEST INFRASTRUCTURE: examples/repair_model.cuh (a machine shop: a repair crew
// cmb_resourcepool and an inspection cmb_resource) compiled for the CPU from the SAME source text twice - on the general engine
// (cimba_b200/csrc/cmb_device.cuh) and on the static tier (cimba_b200/csrc/cmb_static.cuh, cmb::StaticSim<8, 0>) - and
// exported as a small C library, so that tests/test_static_resources.py can hold both to the reference's shop
// (oracle/_ref/librepairdrv.so, tests/golden/repair_vectors.json) trial by trial where there is no GPU.  The CUDA vocabulary
// is mapped to C++ as in tests/cmb_engine_host.cpp.  Not a product path: built by the test, under tests/.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC static_resources_host.cpp -o libstatic_resources_host.so
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

#include "../examples/repair_model.cuh"

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

// engine 0 = the general engine (arena_bytes of growth memory per trial), 1 = the static tier (the shop has no queues, so
// no ring).  trace_cap pops of each trial into trace_key / trace_time [count][trace_cap].  Returns 0, -1 for another engine.
extern "C" int host_repair_run_trials(int engine, int servers, uint64_t master_seed, uint64_t first, uint64_t count,
                                      uint64_t num_objects, double arr_mean, double srv_mean,
                                      const double *params, uint32_t num_params, uint64_t arena_bytes,
                                      uint64_t trace_cap, uint64_t *trace_key, double *trace_time, HostResult *out)
{
    if (engine != 0 && engine != 1) return -1;
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
        in.num_params = num_params;
        for (uint32_t k = 0; k < num_params && k < 16u; k++) in.params[k] = params[k];
        in.trial = first + i;
        const uint64_t seed = fmix64(master_seed, first + i);
        uint64_t *tk = trace_cap ? trace_key + i * trace_cap : nullptr;
        double *tt = trace_cap ? trace_time + i * trace_cap : nullptr;
        cmb::TrialOut o;
        if (engine == 0) {
            unsigned long long cursor = 0;
            cmb::Arena arena{mem.data(), &cursor, arena_bytes};
            cmb::Sim sim;
            repair_example::Repair m;
            sim.init(seed, &hot, arena);
            if (trace_cap) cmb::run_one_trial<repair_example::Repair, true>(sim, m, in, o, trace_cap, tk, tt);
            else           cmb::run_one_trial<repair_example::Repair, false>(sim, m, in, o, 0u, nullptr, nullptr);
            copy_out(sim, o, out[i]);
        }
        else {
            using S = cmb::StaticSim<8, 0>;
            S sim;
            repair_example::RepairT<S> m;
            double win[cmb::STATIC_WINDOW], ring[1];
            sim.init(seed, &hot, win, 1u, ring, 0u);
            cmb::static_run_trial_host(sim, m, in, o, trace_cap, tk, tt);
            copy_out(sim, o, out[i]);
        }
    }
    return 0;
}
