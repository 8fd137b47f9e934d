// capi.cu - the C-ABI shared library (include/cimba_b200.h) over the CUDA engine.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -fmad=false ...
// (see __graft_entry__.build()).  No CPU fallback exists anywhere in this file:
// every compute entry point ends in a kernel launch or fails.
#include <atomic>
#include <chrono>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/cimba_b200.h"
#include "engine.cuh"
#include "queue_model.cuh"
#include "mm1_fast.cuh"
#include "mm1_pc.cuh"
#include "gg1_fast.cuh"
#include "pool_model.cuh"
#include "pool_fast.cuh"
#include "guarded_model.cuh"
#include "preempt_model.cuh"
#include "buffer_model.cuh"
#include "prioq_model.cuh"
#include "timers_model.cuh"
#include "resource_model.cuh"
#include "harbor_model.cuh"
#include "hold_model.cuh"
#include "hold_deep.cuh"
#include "hold_group.cuh"
#include "awacs_model.cuh"
#include "rng.cuh"
#include "distributions.cuh"
#include "summary.cuh"
#include "cmb_launch.cuh"
#include "../models/mm1_model.cuh"
#include "../models/gg1_model.cuh"
#include "../models/mmc_model.cuh"
#include "../models/renege_model.cuh"
#include "../models/hold_general_model.cuh"
#include "../models/cheese_model.cuh"
#include "../models/mm1_recorded_model.cuh"
#include "../models/tutorial1_model.cuh"
#include "../models/park_model.cuh"
#include "../models/tutorial2_model.cuh"
#include "../models/guarded_model.cuh"
#include "../models/workshop_model.cuh"
#include "../models/coverage_models.cuh"
#include "../models/harbor_general_model.cuh"

#include <dlfcn.h>      // cimba_b200_model_load: a model library built with scripts/build_model.py

using namespace cimba_b200;

namespace {

thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

int fail(int code, const char *fmt, const char *detail = "")
{
    snprintf(g_err, sizeof(g_err), fmt, detail);
    return code;
}

int cuda_fail(cudaError_t e, const char *where)
{
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    return CIMBA_B200_ECUDA;
}

#define CUDA_TRY(expr)                                             \
    do {                                                           \
        cudaError_t e_ = (expr);                                   \
        if (e_ != cudaSuccess) return cuda_fail(e_, #expr);        \
    } while (0)

constexpr uint32_t QUEUE_SPILL_CAP = 512u;     // default: doubles per trial behind the 32-entry window

// job.queue_spill_cap: 0 = default, else a power of two up to 2^26; 0xffffffff = invalid
uint32_t spill_cap_of(const cimba_b200_device_job *job)
{
    const uint32_t c = job->queue_spill_cap;
    if (c == 0u) return QUEUE_SPILL_CAP;
    if ((c & (c - 1u)) != 0u || c > (1u << 26)) return 0xffffffffu;
    return c;
}

// ---- the general engine behind the fixed-capacity fast kernels
// A trial the fast M/M/1, G/G/1 or M/M/c kernel had to flag (its queue outgrew window + ring, its event list or wait list
// their fixed tables) is re-run inside the same launch by the general engine, whose containers grow: the reference's
// queue is CMB_UNLIMITED and so is the drop-in.  The repair kernel is enqueued unconditionally behind the fast one and
// looks at the status words; with nothing flagged it costs one pass over them.
constexpr uint32_t REPAIR_BITS = CIMBA_B200_TRIAL_QUEUE_OVERFLOW | CIMBA_B200_TRIAL_FEL_OVERFLOW |
                                 CIMBA_B200_TRIAL_GUARD_OVERFLOW | CIMBA_B200_TRIAL_PROC_OVERFLOW;

uint64_t repair_arena_bytes(const cimba_b200_device_job *job)
{
    uint64_t b = job->num_trials * 32768ull;
    if (b < (64ull << 20)) b = 64ull << 20;
    if (b > (4ull << 30)) b = 4ull << 30;
    return cmb::ARENA_HEADER + b;
}

uint64_t align256(uint64_t v) { return (v + 255u) & ~(uint64_t)255u; }

bool mmc_goes_general(const cimba_b200_device_job *job)
{
    return job->model == CIMBA_B200_MODEL_MMC && (job->variant == CIMBA_B200_VARIANT_GENERAL || job->servers > 14);
}

bool fast_goes_general(const cimba_b200_device_job *job)
{
    return (job->model == CIMBA_B200_MODEL_MM1 || job->model == CIMBA_B200_MODEL_GG1 || job->model == CIMBA_B200_MODEL_MM1_RECORDED) &&
           job->variant == CIMBA_B200_VARIANT_GENERAL;
}

// the tutorial's trial runs on the static tier (two processes, a buffer, three events of its own) unless the general engine is asked for
bool tutorial1_goes_static(const cimba_b200_device_job *job)
{
    return job->model == CIMBA_B200_MODEL_TUTORIAL1 && job->variant != CIMBA_B200_VARIANT_GENERAL;
}

bool goes_static(const cimba_b200_device_job *job)
{
    if (tutorial1_goes_static(job)) return true;
    return (job->model == CIMBA_B200_MODEL_MM1 || job->model == CIMBA_B200_MODEL_GG1 || job->model == CIMBA_B200_MODEL_MM1_RECORDED) &&
           job->variant == CIMBA_B200_VARIANT_STATIC;
}

bool hold_goes_general(const cimba_b200_device_job *job)
{
    return job->model == CIMBA_B200_MODEL_HOLD && job->variant == CIMBA_B200_VARIANT_GENERAL;
}

bool harbor_goes_general(const cimba_b200_device_job *job)
{
    return job->model == CIMBA_B200_MODEL_HARBOR && job->variant == CIMBA_B200_VARIANT_GENERAL;
}

// models loaded with cimba_b200_model_load
struct UserModel {
    void *handle;
    std::string name;
    uint64_t (*workspace_bytes)(const cimba_b200_device_job *);
    int (*launch)(const cimba_b200_device_job *, void *);
};
std::mutex g_user_mu;
std::deque<UserModel> g_user_models;          // a deque: loaded models never move

const UserModel *user_model(int id)
{
    std::lock_guard<std::mutex> hold(g_user_mu);
    const int k = id - CIMBA_B200_MODEL_USER_BASE;
    return (k >= 0 && (size_t)k < g_user_models.size()) ? &g_user_models[(size_t)k] : nullptr;
}

template <class Model>
int launch_general(const cimba_b200_device_job *job, unsigned char *arena, uint64_t bytes, uint32_t only_flagged, cudaStream_t st,
                   const char *what)
{
    const int e = cmb::launch_model<Model>(*job, arena, bytes, only_flagged, st);
    g_launches++;
    return e == 0 ? CIMBA_B200_OK : cuda_fail((cudaError_t)e, what);
}

// the reference's own test worlds (models 3-6, 8, 11-14): like M/M/1, G/G/1 and M/M/c they have a fixed-capacity kernel
// (csrc/general.cuh, faster than the engine) behind which the general engine re-runs whatever that
// kernel flags; a capacity its tables cannot hold, or CIMBA_B200_VARIANT_GENERAL, goes to the engine directly
bool coverage_goes_general(const cimba_b200_device_job *job);

template <template <class> class F, class... A>
auto for_coverage_model(int model, A &&...a)
{
    switch (model) {
    case CIMBA_B200_MODEL_GUARDED:           return F<models::Guarded<false, false>>::call(a...);
    case CIMBA_B200_MODEL_GUARDED_RECORDED:  return F<models::Guarded<false, true>>::call(a...);
    case CIMBA_B200_MODEL_PRIOQ_RECORDED:    return F<models::Guarded<true, true>>::call(a...);
    case CIMBA_B200_MODEL_PREEMPT:           return F<models::PoolFight>::call(a...);
    case CIMBA_B200_MODEL_BUFFER:            return F<models::Workshop<false>>::call(a...);
    case CIMBA_B200_MODEL_BUFFER_RECORDED:   return F<models::Workshop<true>>::call(a...);
    case CIMBA_B200_MODEL_PRIOQ:             return F<models::QueueAndTide>::call(a...);
    case CIMBA_B200_MODEL_TIMERS:            return F<models::FrontDesk>::call(a...);
    default:                                 return F<models::Tool>::call(a...);       // CIMBA_B200_MODEL_RESOURCE_RECORDED
    }
}

template <class Model>
struct WorkspaceOf {
    static uint64_t call(const cimba_b200_device_job *job) { return cmb::workspace_bytes_for<Model>(*job); }
};

bool is_queue_model(int m)
{
    return m == CIMBA_B200_MODEL_MM1 || m == CIMBA_B200_MODEL_GG1 || m == CIMBA_B200_MODEL_MM1_RECORDED;
}
#ifndef HOLD_DEFAULT_LANES
#define HOLD_DEFAULT_LANES 32      // lanes per trial of the default hold kernel (H100, 4096 trials x 1000 workers: 32 -> 304 ms, 16 -> 415, 8 -> 745)
#endif

// spill area of one warp of hold_deep_kernel: the heap nodes below level 1, whole rows of 32
uint64_t deep_row_entries(int workers)
{
    const uint64_t count = (uint64_t)(workers < 1 ? 1 : workers) + 2u;
    const uint64_t below = count > 33u ? count - 33u : 0u;
    return ((below + 31u) / 32u) * 32u + 32u;
}

bool is_general_model(int m)
{
    return m == CIMBA_B200_MODEL_GUARDED || m == CIMBA_B200_MODEL_PREEMPT || m == CIMBA_B200_MODEL_BUFFER ||
           m == CIMBA_B200_MODEL_PRIOQ || m == CIMBA_B200_MODEL_TIMERS || m == CIMBA_B200_MODEL_GUARDED_RECORDED ||
           m == CIMBA_B200_MODEL_BUFFER_RECORDED || m == CIMBA_B200_MODEL_PRIOQ_RECORDED ||
           m == CIMBA_B200_MODEL_RESOURCE_RECORDED;
}

bool coverage_goes_general(const cimba_b200_device_job *job)
{
    if (!is_general_model(job->model)) return false;
    if (job->variant == CIMBA_B200_VARIANT_GENERAL) return true;
    const int m = job->model;
    if (m == CIMBA_B200_MODEL_TIMERS || m == CIMBA_B200_MODEL_RESOURCE_RECORDED || m == CIMBA_B200_MODEL_PREEMPT ||
        m == CIMBA_B200_MODEL_BUFFER || m == CIMBA_B200_MODEL_BUFFER_RECORDED) return false;      // no table sized by `servers`
    return job->servers > ((m == CIMBA_B200_MODEL_PRIOQ || m == CIMBA_B200_MODEL_PRIOQ_RECORDED) ? 15 : 16);
}

template <class Model>
struct LaunchOf {
    static int call(const cimba_b200_device_job *job, unsigned char *arena, uint64_t bytes, uint32_t only_flagged, cudaStream_t st)
    {
        return launch_general<Model>(job, arena, bytes, only_flagged, st, only_flagged ? "repair pass" : "trial_kernel launch");
    }
};

// ---------------------------------------------------------------- RNG KAT kernel
__global__ void rng_draws_kernel(uint64_t seed, int kind, double p0, double p1, uint64_t n, double *out)
{
    __shared__ ZigHot hot;
    stage_zig_hot(hot, true);
    __syncthreads();
    if (threadIdx.x != 0 || blockIdx.x != 0) {
        return;
    }
    Sfc64 r;
    r.seed(seed);
    for (uint64_t i = 0; i < n; i++) {
        double v = 0.0;
        switch (kind) {
        case 0: v = __longlong_as_double((long long)r.next()); break;
        case 1: v = r.exponential(hot, p0); break;
        case 2: v = r.std_normal(hot); break;
        case 3: v = r.uniform01(); break;
        case 4: v = r.normal(hot, p0, p1); break;
        case 5: v = r.erlang(hot, (unsigned)p0, p1); break;
        case 6: v = r.uniform(p0, p1); break;
        case 7: v = (double)r.dice((long long)p0, (long long)p1); break;
        case 8: v = (double)r.bernoulli(p0); break;
        }
        out[i] = v;
    }
}

struct DrawParams {
    double   v[CIMBA_B200_RNG_MAX_PARAMS];
    uint64_t uprob[CIMBA_B200_RNG_MAX_PARAMS];
    uint32_t alias[CIMBA_B200_RNG_MAX_PARAMS];
};

__global__ void rng_draws_ex_kernel(uint64_t seed, int kind, const DrawParams par, uint64_t n, double *out)
{
    __shared__ ZigHot hot;
    stage_zig_hot(hot, true);
    __syncthreads();
    if (threadIdx.x != 0 || blockIdx.x != 0) {
        return;
    }
    Sfc64 r;
    r.seed(seed);
    FlipCache flips{0u, 0u};
    const double *p = par.v;
    const unsigned cnt = (unsigned)p[0];
    for (uint64_t i = 0; i < n; i++) {
        double v = 0.0;
        switch (kind) {
        case 9:  v = rnd_triangular(r, p[0], p[1], p[2]); break;
        case 10: v = rnd_lognormal(r, hot, p[0], p[1]); break;
        case 11: v = rnd_logistic(r, p[0], p[1]); break;
        case 12: v = rnd_cauchy(r, hot, p[0], p[1]); break;
        case 13: v = rnd_hypoexponential(r, hot, cnt, p + 1); break;
        case 14: v = rnd_hyperexponential(r, hot, cnt, p + 1, p + 1 + cnt); break;
        case 15: v = rnd_gamma(r, hot, p[0], p[1]); break;
        case 16: v = rnd_beta(r, hot, p[0], p[1], p[2], p[3]); break;
        case 17: v = rnd_PERT_mod(r, hot, p[0], p[1], p[2], 4.0); break;
        case 18: v = rnd_weibull(r, hot, p[0], p[1]); break;
        case 19: v = rnd_pareto(r, p[0], p[1]); break;
        case 20: v = rnd_chisquared(r, hot, p[0]); break;
        case 21: v = rnd_F_dist(r, hot, p[0], p[1]); break;
        case 22: v = rnd_t_dist(r, hot, p[0], p[1], p[2]); break;
        case 23: v = rnd_rayleigh(r, hot, p[0]); break;
        case 24: v = (double)rnd_flip(r, flips); break;
        case 25: v = (double)rnd_geometric(r, hot, p[0]); break;
        case 26: v = (double)rnd_binomial(r, cnt, p[1]); break;
        case 27: v = (double)rnd_negative_binomial(r, hot, cnt, p[1]); break;
        case 28: v = (double)rnd_poisson(r, hot, p[0]); break;
        case 29: v = (double)rnd_loaded_dice(r, cnt, p + 1); break;
        case 30: v = (double)rnd_alias_sample(r, cnt, par.uprob, par.alias); break;
        case 31: v = rnd_std_gamma(r, hot, p[0]); break;
        case 32: v = rnd_PERT_mod(r, hot, p[0], p[1], p[2], p[3]); break;
        case 33: v = (double)rnd_negative_binomial(r, hot, cnt, p[1]); break;
        }
        out[i] = v;
    }
}

uint64_t alias_secure(double p)        // src/cmb_random.c:672-686
{
    if (p <= 0.0) return 0u;
    if (p >= 1.0) return UINT64_MAX;
    return (uint64_t)(p * (double)UINT64_MAX);
}

// ---------------------------------------------------------------- MODEL_AWACS host side
constexpr int MAX_TERRAIN_DEVICES = 64;
std::mutex g_terrain_mu;
AwacsTerrain g_terrain[MAX_TERRAIN_DEVICES];
bool g_terrain_set[MAX_TERRAIN_DEVICES];
float *g_terrain_owned[MAX_TERRAIN_DEVICES];     // device copies made by cimba_b200_awacs_upload_terrain
float *g_terrain_tiles[MAX_TERRAIN_DEVICES];     // tile-maximum maps (aw_tile_max_kernel), always library-owned

// racetrack_initialize with run_trial's arguments (tutorial/tut_5_1.c:724-782, :1177-1188): constants of the
// model, evaluated once on the host with the host's libm, exactly as the reference evaluates them
AwacsOrbit awacs_orbit()
{
    const double PI = 3.14159265358979323846;
    const double deg_to_rad = (2.0 * PI / 360.0), nm_to_meters = 1852.0, feet_to_meters = 0.3048;
    const double knots_to_ms = (1852.0 / 3600.0);
    const double WGS84_A = 6378137.0, WGS84_F = (1.0 / 298.257223563), WGS84_E2 = (WGS84_F * (2.0 - WGS84_F));
    const float start_time = 0.0f, anchor_lat = 30.0f, orientation = 0.0f, leg_length = 50.0f;
    const float turn_radius = 10.0f, flight_level = 310.0f, velocity = 300.0f;
    AwacsOrbit o{};
    o.start_time = 3600.0f * start_time;
    const float anchor_lat_r = (float)(anchor_lat * deg_to_rad);
    o.orientation_r = (float)((90.0 - orientation) * deg_to_rad);
    o.length_m = (float)(leg_length * nm_to_meters);
    o.turn_radius_m = (float)(turn_radius * nm_to_meters);
    o.altitude_m = (float)(flight_level * 100.0 * feet_to_meters);
    o.velocity_ms = (float)(velocity * knots_to_ms);
    o.turn_dist_m = (float)(PI * o.turn_radius_m);
    o.orbit_dist_m = 2.0f * (o.length_m + o.turn_dist_m);
    o.side = -1.0f;                                     // clockwise
    const double sin_lat = sinf(anchor_lat_r);
    const double common = 1.0 - (WGS84_E2 * sin_lat * sin_lat);
    const double sqrt_common = sqrt(common);
    const double M = WGS84_A * (1.0 - WGS84_E2) / (common * sqrt_common);
    const double N = WGS84_A / sqrt_common;
    const double g = 9.80665;
    const double roll_mag = atan((o.velocity_ms * o.velocity_ms) / (o.turn_radius_m * g));
    o.roll_angle_r = (float)(roll_mag * -o.side);
    o.rad_eff = (float)(sqrt(M * N) * (4.0 / 3.0));
    o.cos_o = cos((double)o.orientation_r);
    o.sin_o = sin((double)o.orientation_r);
    return o;
}

template <int MODEL>
int launch_queue(const QueueArgs &qa, bool trace, dim3 grid, cudaStream_t st)
{
    if (trace) {
        queue_kernel<MODEL, true><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
    }
    else {
        queue_kernel<MODEL, false><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
    }
    g_launches++;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "queue_kernel launch");
}

}  // namespace

extern "C" {

const char *cimba_b200_version(void) { return CIMBA_B200_VERSION_STRING; }
const char *cimba_b200_last_error(void) { return g_err; }
uint64_t cimba_b200_launch_count(void) { return g_launches.load(); }
uint64_t cimba_b200_fmix64(uint64_t seed, uint64_t nonce) { return fmix64(seed, nonce); }

int cimba_b200_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        (void)cudaGetLastError();
        return 0;
    }
    return n;
}

uint64_t cimba_b200_workspace_bytes(const cimba_b200_device_job *job)
{
    if (job == nullptr) {
        return 0u;
    }
    if (job->model >= CIMBA_B200_MODEL_USER_BASE) {
        const UserModel *um = user_model(job->model);
        return um ? um->workspace_bytes(job) : 0u;
    }
    if (job->model == CIMBA_B200_MODEL_RENEGE) return cmb::workspace_bytes_for<models::Renege>(*job);
    if (job->model == CIMBA_B200_MODEL_POOL_RECORDED) return cmb::workspace_bytes_for<models::Cheese>(*job);
    if (job->model == CIMBA_B200_MODEL_PARK) return cmb::workspace_bytes_for<models::Park>(*job);
    if (job->model == CIMBA_B200_MODEL_TUTORIAL2) return cmb::workspace_bytes_for<models::Tutorial2>(*job);
    if (job->model == CIMBA_B200_MODEL_TUTORIAL1 && !tutorial1_goes_static(job)) return cmb::workspace_bytes_for<models::Tutorial1>(*job);
    if (coverage_goes_general(job)) return for_coverage_model<WorkspaceOf>(job->model, job);
    if (mmc_goes_general(job)) return cmb::workspace_bytes_for<models::MMC>(*job);
    if (hold_goes_general(job)) return cmb::workspace_bytes_for<models::HoldGeneral>(*job);
    if (harbor_goes_general(job)) return cmb::workspace_bytes_for<models::HarborGeneral>(*job);
    if (goes_static(job)) {
        if (job->model == CIMBA_B200_MODEL_TUTORIAL1) return cmb::workspace_bytes_static<models::Tutorial1T, 2, 0, 3>(*job);
        return job->model == CIMBA_B200_MODEL_MM1 ? cmb::workspace_bytes_static<models::MM1T, 2, 1>(*job)
             : job->model == CIMBA_B200_MODEL_GG1 ? cmb::workspace_bytes_static<models::GG1T, 2, 1>(*job)
                                                  : cmb::workspace_bytes_static<models::MM1RecordedT, 2, 1>(*job);
    }
    if (fast_goes_general(job)) {
        return job->model == CIMBA_B200_MODEL_MM1 ? cmb::workspace_bytes_for<models::MM1>(*job)
             : job->model == CIMBA_B200_MODEL_GG1 ? cmb::workspace_bytes_for<models::GG1>(*job)
                                                  : cmb::workspace_bytes_for<models::MM1Recorded>(*job);
    }
    if (is_queue_model(job->model) || job->model == CIMBA_B200_MODEL_MMC) {
        const uint32_t cap = spill_cap_of(job);
        const uint64_t rings = job->num_trials * (uint64_t)(cap == 0xffffffffu ? QUEUE_SPILL_CAP : cap) * sizeof(double);
        // the rings of the fast kernel, then the growth arena of its repair pass
        return align256(rings) + repair_arena_bytes(job);
    }
    if (job->model == CIMBA_B200_MODEL_HARBOR) {
        return job->num_trials * (uint64_t)sizeof(HarborState);
    }
    if (job->model == CIMBA_B200_MODEL_HOLD && job->variant != 1) {
        return job->num_trials * deep_row_entries(job->servers) * (uint64_t)sizeof(uint4);
    }
    if (job->model == CIMBA_B200_MODEL_AWACS) {
        return job->num_trials * (uint64_t)AWACS_STATE_BYTES;
    }
    if (is_general_model(job->model)) {
        return align256(job->num_trials * (uint64_t)sizeof(GeneralState)) + repair_arena_bytes(job);
    }
    return 0u;
}

int cimba_b200_launch(const cimba_b200_device_job *job, void *stream)
{
    if (job == nullptr) return fail(CIMBA_B200_EINVAL, "job is NULL");
    if (job->num_trials == 0u) return fail(CIMBA_B200_EINVAL, "num_trials must be > 0 (src/cimba.c:157)");
    if ((job->arr_mean == nullptr || job->srv_mean == nullptr) && job->model != CIMBA_B200_MODEL_AWACS)
        return fail(CIMBA_B200_EINVAL, "arr_mean/srv_mean device arrays are required");
    if (job->num_objects >= 0xffffffffull) return fail(CIMBA_B200_EINVAL, "num_objects must be < 2^32-1");
    const int mapping = job->mapping == 0 ? CIMBA_B200_MAP_LANE : job->mapping;
    if (mapping != CIMBA_B200_MAP_LANE && mapping != CIMBA_B200_MAP_WARP)
        return fail(CIMBA_B200_EINVAL, "mapping must be CIMBA_B200_MAP_LANE or CIMBA_B200_MAP_WARP");
    const bool trace = job->trace_cap > 0u;
    if (trace && (job->trace_key == nullptr || job->trace_time == nullptr))
        return fail(CIMBA_B200_EINVAL, "trace_cap > 0 needs trace_key and trace_time");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    cudaStream_t st = (cudaStream_t)stream;
    if (spill_cap_of(job) == 0xffffffffu)
        return fail(CIMBA_B200_EINVAL, "queue_spill_cap must be 0 (default) or a power of two <= 2^26");
    if (job->num_params > CIMBA_B200_MAX_MODEL_PARAMS || (job->num_params > 0u && job->params == nullptr))
        return fail(CIMBA_B200_EINVAL, "params: at most CIMBA_B200_MAX_MODEL_PARAMS doubles behind a HOST pointer");

    if (job->model >= CIMBA_B200_MODEL_USER_BASE) {
        const UserModel *um = user_model(job->model);
        if (um == nullptr) return fail(CIMBA_B200_EINVAL, "unknown model id (cimba_b200_model_load returns the ids of loaded models)");
        if (job->workspace_bytes < um->workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        const int e = um->launch(job, stream);
        g_launches++;
        return e == 0 ? CIMBA_B200_OK : cuda_fail((cudaError_t)e, um->name.c_str());
    }
    if (goes_static(job)) {
        if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "the static tier runs one trial per lane (CIMBA_B200_MAP_LANE)");
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        const int e = job->model == CIMBA_B200_MODEL_TUTORIAL1 ? cmb::launch_static_model<models::Tutorial1T, 2, 0, 3>(*job, st)
                    : job->model == CIMBA_B200_MODEL_MM1 ? cmb::launch_static_model<models::MM1T, 2, 1>(*job, st)
                    : job->model == CIMBA_B200_MODEL_GG1 ? cmb::launch_static_model<models::GG1T, 2, 1>(*job, st)
                                                         : cmb::launch_static_model<models::MM1RecordedT, 2, 1>(*job, st);
        g_launches += job->status != nullptr ? 2 : 1;
        return e == 0 ? CIMBA_B200_OK : cuda_fail((cudaError_t)e, "static_trial_kernel launch");
    }
    if (coverage_goes_general(job)) {
        if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "the general engine runs one trial per lane (CIMBA_B200_MAP_LANE)");
        const bool no_capacity = job->model == CIMBA_B200_MODEL_TIMERS || job->model == CIMBA_B200_MODEL_RESOURCE_RECORDED;
        if (!no_capacity && job->servers < 1) return fail(CIMBA_B200_EINVAL, "capacity (servers) must be >= 1");
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        return for_coverage_model<LaunchOf>(job->model, job, (unsigned char *)job->workspace, job->workspace_bytes, 0u, st);
    }
    if (job->model == CIMBA_B200_MODEL_RENEGE || job->model == CIMBA_B200_MODEL_POOL_RECORDED || job->model == CIMBA_B200_MODEL_TUTORIAL1 || job->model == CIMBA_B200_MODEL_PARK || job->model == CIMBA_B200_MODEL_TUTORIAL2 || mmc_goes_general(job) || fast_goes_general(job) || hold_goes_general(job) || harbor_goes_general(job)) {
        if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "the general engine runs one trial per lane (CIMBA_B200_MAP_LANE)");
        if (job->servers < 1) return fail(CIMBA_B200_EINVAL, "servers must be >= 1");
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        unsigned char *ws = (unsigned char *)job->workspace;
        if (job->model == CIMBA_B200_MODEL_RENEGE)
            return launch_general<models::Renege>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<Renege> launch");
        if (job->model == CIMBA_B200_MODEL_TUTORIAL2)
            return launch_general<models::Tutorial2>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<Tutorial2> launch");
        if (job->model == CIMBA_B200_MODEL_PARK)
            return launch_general<models::Park>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<Park> launch");
        if (job->model == CIMBA_B200_MODEL_TUTORIAL1)
            return launch_general<models::Tutorial1>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<Tutorial1> launch");
        if (job->model == CIMBA_B200_MODEL_POOL_RECORDED)
            return launch_general<models::Cheese>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<Cheese> launch");
        if (job->model == CIMBA_B200_MODEL_MMC)
            return launch_general<models::MMC>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<MMC> launch");
        if (job->model == CIMBA_B200_MODEL_HOLD)
            return launch_general<models::HoldGeneral>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<HoldGeneral> launch");
        if (job->model == CIMBA_B200_MODEL_HARBOR) {
            if (job->servers < 3) return fail(CIMBA_B200_EINVAL, "tugs (servers) must be >= 3 for CIMBA_B200_MODEL_HARBOR (a large ship needs 3)");
            return launch_general<models::HarborGeneral>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<HarborGeneral> launch");
        }
        if (job->model == CIMBA_B200_MODEL_MM1)
            return launch_general<models::MM1>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<MM1> launch");
        if (job->model == CIMBA_B200_MODEL_MM1_RECORDED)
            return launch_general<models::MM1Recorded>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<MM1Recorded> launch");
        return launch_general<models::GG1>(job, ws, job->workspace_bytes, 0u, st, "trial_kernel<GG1> launch");
    }

    if (is_queue_model(job->model)) {
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        QueueArgs qa{};
        qa.mapping = mapping;
        qa.master_seed = job->master_seed;
        qa.first_trial = job->first_trial;
        qa.num_trials = job->num_trials;
        qa.num_objects = job->num_objects;
        qa.arr_mean = job->arr_mean;
        qa.srv_mean = job->srv_mean;
        qa.events = job->events;
        qa.objects = job->objects;
        qa.t_end = job->t_end;
        qa.sum_wait = job->sum_wait;
        qa.status = job->status;
        qa.max_queue = job->max_queue;
        qa.counters = job->counters;
        qa.spill = (double *)job->workspace;
        qa.spill_cap = spill_cap_of(job);
        qa.trace_cap = job->trace_cap;
        qa.trace_key = job->trace_key;
        qa.trace_time = job->trace_time;
        qa.diag = (unsigned long long *)job->diag;
        const uint64_t threads = job->num_trials * (uint64_t)mapping;
        const uint64_t blocks = (threads + QUEUE_BLOCK - 1) / QUEUE_BLOCK;
        if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
        dim3 grid((unsigned)blocks);
        if (job->model == CIMBA_B200_MODEL_GG1) {
            if (job->variant == 1) return launch_queue<1>(qa, trace, grid, st);
            if (trace) gg1_kernel<true><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
            else       gg1_kernel<false><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
            g_launches++;
            cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return cuda_fail(e, "gg1_kernel launch");
            if (job->status == nullptr) return CIMBA_B200_OK;       // nobody could see a flag: nothing to repair by
            return launch_general<models::GG1>(job, (unsigned char *)job->workspace + align256(job->num_trials * (uint64_t)qa.spill_cap * sizeof(double)),
                                               repair_arena_bytes(job), REPAIR_BITS, st, "repair pass (G/G/1)");
        }
        if (job->model == CIMBA_B200_MODEL_MM1_RECORDED) {
            if (job->counters == nullptr)
                return fail(CIMBA_B200_EINVAL, "CIMBA_B200_MODEL_MM1_RECORDED writes its cmb_wtdsummary to counters[]");
            if (trace) queue_kernel<0, true, true><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
            else       queue_kernel<0, false, true><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
            g_launches++;
            cudaError_t e = cudaGetLastError();
            if (e != cudaSuccess) return cuda_fail(e, "queue_kernel (recorded) launch");
            if (job->status == nullptr) return CIMBA_B200_OK;
            return launch_general<models::MM1Recorded>(job, (unsigned char *)job->workspace + align256(job->num_trials * (uint64_t)qa.spill_cap * sizeof(double)),
                                                       repair_arena_bytes(job), REPAIR_BITS, st, "repair pass (M/M/1 with its queue history)");
        }
        if (job->variant == 1) return launch_queue<0>(qa, trace, grid, st);
        if (job->variant == 2) {                        // variates from producer warps (mm1_pc.cuh): an experiment, same answers
            if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "variant 2 of MODEL_MM1 runs one trial per lane");
            const dim3 pc_grid((unsigned)((job->num_trials + MM1_PC_CONSUMERS - 1) / MM1_PC_CONSUMERS));
            if (trace) mm1_pc_kernel<true><<<pc_grid, 2 * MM1_PC_CONSUMERS, 0, st>>>(qa);
            else       mm1_pc_kernel<false><<<pc_grid, 2 * MM1_PC_CONSUMERS, 0, st>>>(qa);
        }
        else if (trace) {
            mm1_kernel<true><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
        }
        else {
            mm1_kernel<false><<<grid, QUEUE_BLOCK, 0, st>>>(qa);
        }
        g_launches++;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_fail(e, "mm1_kernel launch");
        if (job->status == nullptr) return CIMBA_B200_OK;           // nobody could see a flag: nothing to repair by
        return launch_general<models::MM1>(job, (unsigned char *)job->workspace + align256(job->num_trials * (uint64_t)qa.spill_cap * sizeof(double)),
                                           repair_arena_bytes(job), REPAIR_BITS, st, "repair pass (M/M/1)");
    }
    if (job->model == CIMBA_B200_MODEL_MMC) {
        if (job->servers < 1) return fail(CIMBA_B200_EINVAL, "servers must be >= 1 for CIMBA_B200_MODEL_MMC");
        if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "MODEL_MMC supports CIMBA_B200_MAP_LANE only");
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        PoolArgs pa{};
        pa.servers = job->servers;
        pa.master_seed = job->master_seed;
        pa.first_trial = job->first_trial;
        pa.num_trials = job->num_trials;
        pa.num_objects = job->num_objects;
        pa.arr_mean = job->arr_mean;
        pa.srv_mean = job->srv_mean;
        pa.events = job->events;
        pa.objects = job->objects;
        pa.t_end = job->t_end;
        pa.sum_wait = job->sum_wait;
        pa.status = job->status;
        pa.max_queue = job->max_queue;
        pa.spill = (double *)job->workspace;
        pa.spill_cap = spill_cap_of(job);
        pa.trace_cap = job->trace_cap;
        pa.trace_key = job->trace_key;
        pa.trace_time = job->trace_time;
        pa.diag = (unsigned long long *)job->diag;
        const uint64_t blocks = (job->num_trials + POOL_BLOCK - 1) / POOL_BLOCK;
        if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
        if (job->variant == 1) {                        // the readable formulation, pool_model.cuh
            if (trace) pool_kernel<true><<<(unsigned)blocks, POOL_BLOCK, 0, st>>>(pa);
            else       pool_kernel<false><<<(unsigned)blocks, POOL_BLOCK, 0, st>>>(pa);
        }
        else if (trace) {
            pool_fast_kernel<true><<<(unsigned)blocks, POOL_BLOCK, 0, st>>>(pa);
        }
        else {
            pool_fast_kernel<false><<<(unsigned)blocks, POOL_BLOCK, 0, st>>>(pa);
        }
        g_launches++;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_fail(e, "pool_kernel launch");
        if (job->status == nullptr) return CIMBA_B200_OK;
        return launch_general<models::MMC>(job, (unsigned char *)job->workspace + align256(job->num_trials * (uint64_t)pa.spill_cap * sizeof(double)),
                                           repair_arena_bytes(job), REPAIR_BITS, st, "repair pass (M/M/c)");
    }
    if (is_general_model(job->model)) {
        const bool rsc = job->model == CIMBA_B200_MODEL_RESOURCE_RECORDED;
        const bool tmr = job->model == CIMBA_B200_MODEL_TIMERS || rsc;      // no capacity argument
        const bool prq = job->model == CIMBA_B200_MODEL_PRIOQ;
        const bool pre = job->model == CIMBA_B200_MODEL_PREEMPT;
        const bool buf = job->model == CIMBA_B200_MODEL_BUFFER || job->model == CIMBA_B200_MODEL_BUFFER_RECORDED;
        const bool pq13 = job->model == CIMBA_B200_MODEL_PRIOQ_RECORDED;
        if (!tmr && job->servers < 1) return fail(CIMBA_B200_EINVAL, "capacity (servers) must be >= 1");
        if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "MODEL_GUARDED supports CIMBA_B200_MAP_LANE only");
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        GuardedArgs ga{};
        ga.capacity = job->servers;
        ga.master_seed = job->master_seed;
        ga.first_trial = job->first_trial;
        ga.num_trials = job->num_trials;
        ga.duration = job->num_objects;
        ga.put_mean = job->arr_mean;
        ga.get_mean = job->srv_mean;
        ga.events = job->events;
        ga.objects = job->objects;
        ga.t_end = job->t_end;
        ga.sum_wait = job->sum_wait;
        ga.status = job->status;
        ga.max_queue = job->max_queue;
        ga.counters = job->counters;
        ga.state = (GeneralState *)job->workspace;
        ga.record = (job->model == CIMBA_B200_MODEL_GUARDED_RECORDED || job->model == CIMBA_B200_MODEL_BUFFER_RECORDED ||
                     job->model == CIMBA_B200_MODEL_PRIOQ_RECORDED) ? 1u : 0u;
        ga.use_pq = job->model == CIMBA_B200_MODEL_PRIOQ_RECORDED ? 1u : 0u;
        ga.trace_cap = job->trace_cap;
        ga.trace_key = job->trace_key;
        ga.trace_time = job->trace_time;
        const uint64_t blocks = (job->num_trials + GUARDED_BLOCK - 1) / GUARDED_BLOCK;
        if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
        if (rsc) {
            if (trace) resource_kernel<true><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
            else       resource_kernel<false><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
        }
        else if (tmr) {
            if (trace) timers_kernel<true><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
            else       timers_kernel<false><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
        }
        else if (prq) {
            if (trace) prioq_kernel<true><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
            else       prioq_kernel<false><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
        }
        else if (buf) {
            if (trace) buffer_kernel<true><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
            else       buffer_kernel<false><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
        }
        else if (pre) {
            if (trace) preempt_kernel<true><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
            else       preempt_kernel<false><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
        }
        else if (trace) {
            guarded_kernel<true><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
        }
        else {
            guarded_kernel<false><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ga);
        }
        g_launches++;
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return cuda_fail(e, "guarded_kernel launch");
        if (job->status == nullptr) return CIMBA_B200_OK;
        return for_coverage_model<LaunchOf>(job->model, job, (unsigned char *)job->workspace + align256(job->num_trials * (uint64_t)sizeof(GeneralState)),
                                            repair_arena_bytes(job), REPAIR_BITS, st);
    }
    if (job->model == CIMBA_B200_MODEL_HARBOR) {
        if (job->servers < 3 || job->servers > 255)
            return fail(CIMBA_B200_EINVAL, "tugs (servers) must be in 3..255 for CIMBA_B200_MODEL_HARBOR (a large ship needs 3)");
        if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "MODEL_HARBOR supports CIMBA_B200_MAP_LANE only");
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        HarborArgs ha{};
        ha.tugs = job->servers;
        ha.master_seed = job->master_seed;
        ha.first_trial = job->first_trial;
        ha.num_trials = job->num_trials;
        ha.duration = job->num_objects;
        ha.arr_mean = job->arr_mean;
        ha.unload_small = job->srv_mean;
        ha.events = job->events;
        ha.objects = job->objects;
        ha.t_end = job->t_end;
        ha.sum_wait = job->sum_wait;
        ha.status = job->status;
        ha.max_queue = job->max_queue;
        ha.counters = job->counters;
        ha.state = job->workspace;
        ha.trace_cap = job->trace_cap;
        ha.trace_key = job->trace_key;
        ha.trace_time = job->trace_time;
        // variant 0: up to 32 768 trials run warp-per-trial with the state in shared memory, and whatever trial
        // outgrew those tables is re-run by the lane-per-trial kernel with the large HBM-resident tables; more
        // trials go lane-per-trial directly.  (H100, 400 W, 600 h per trial: warp-per-trial 44 / 154 / 299 ms
        // at 4096 / 16 384 / 32 768 trials, lane-per-trial 151 / 200 / 406 ms.)
        // variant 1 = warp-per-trial only (overflow -> status), variant 2 = lane-per-trial only.
        const bool on_chip_first = job->variant == 1 ||
                                   (job->variant == 0 && job->num_trials <= 32768u && job->status != nullptr);
        ha.repair = 0u;
        if (on_chip_first) {
            const size_t smem = (HARBOR_BLOCK_ON_CHIP / 32) * sizeof(HarborStateOnChip);
            const void *fn = trace ? (const void *)harbor_on_chip_kernel<true> : (const void *)harbor_on_chip_kernel<false>;
            CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int dev = 0, sms = 132, per_sm = 0;
            CUDA_TRY(cudaGetDevice(&dev));
            CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
            cudaError_t oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, HARBOR_BLOCK_ON_CHIP, smem);
            if (oe != cudaSuccess || per_sm < 1) per_sm = 4;
            const uint64_t per_block = HARBOR_BLOCK_ON_CHIP / 32;
            const uint64_t resident = (uint64_t)sms * (uint64_t)per_sm;
            const uint64_t wanted = (job->num_trials + per_block - 1) / per_block;
            const unsigned nb = (unsigned)(wanted < resident ? wanted : resident);
            void *kargs[] = { (void *)&ha };
            cudaError_t le = cudaLaunchKernel(fn, dim3(nb), dim3(HARBOR_BLOCK_ON_CHIP), kargs, smem, st);
            g_launches++;
            cudaError_t e2 = le != cudaSuccess ? le : cudaGetLastError();
            if (e2 != cudaSuccess) return cuda_fail(e2, "harbor_on_chip_kernel launch");
            if (job->variant == 1) return CIMBA_B200_OK;
            ha.repair = 1u;
        }
        const uint64_t blocks = (job->num_trials + GUARDED_BLOCK - 1) / GUARDED_BLOCK;
        if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
        if (trace) harbor_kernel<true><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ha);
        else       harbor_kernel<false><<<(unsigned)blocks, GUARDED_BLOCK, 0, st>>>(ha);
        g_launches++;
        cudaError_t e = cudaGetLastError();
        return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "harbor_kernel launch");
    }
    if (job->model == CIMBA_B200_MODEL_AWACS) {
        if (job->num_objects == 0u) return fail(CIMBA_B200_EINVAL, "MODEL_AWACS: num_objects = trial duration in seconds, > 0");
        if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
            return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
        int dev = 0;
        CUDA_TRY(cudaGetDevice(&dev));
        AwacsArgs aa{};
        {
            std::lock_guard<std::mutex> hold(g_terrain_mu);
            if (dev < 0 || dev >= MAX_TERRAIN_DEVICES || !g_terrain_set[dev])
                return fail(CIMBA_B200_EINVAL, "MODEL_AWACS: no terrain registered on this device; call cimba_b200_awacs_set_terrain()");
            aa.ter = g_terrain[dev];
        }
        aa.orbit = awacs_orbit();
        aa.master_seed = job->master_seed;
        aa.first_trial = job->first_trial;
        aa.num_trials = job->num_trials;
        aa.t_end_s = (double)job->num_objects;
        aa.state = (unsigned char *)job->workspace;
        aa.events = job->events;
        aa.objects = job->objects;
        aa.t_end = job->t_end;
        aa.sum_wait = job->sum_wait;
        aa.status = job->status;
        aa.max_queue = job->max_queue;
        aa.counters = job->counters;
        aa.trace_cap = job->trace_cap;
        aa.trace_key = job->trace_key;
        aa.trace_time = job->trace_time;
        const uint64_t per_block = AWACS_BLOCK / 32;
        const uint64_t blocks = (job->num_trials + per_block - 1) / per_block;
        if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
        if (trace) awacs_kernel<true><<<(unsigned)blocks, AWACS_BLOCK, 0, st>>>(aa);
        else       awacs_kernel<false><<<(unsigned)blocks, AWACS_BLOCK, 0, st>>>(aa);
        g_launches++;
        cudaError_t e = cudaGetLastError();
        return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "awacs_kernel launch");
    }
    if (job->model == CIMBA_B200_MODEL_HOLD) {
        const bool on_chip = job->variant == 1;         // hold_model.cuh: the whole list in shared memory
        if (job->servers < 1 || (on_chip && job->servers > HOLD_CAP - 8) ||
            (uint32_t)job->servers + 2u > DEEP_MAX_ENTRIES)
            return fail(CIMBA_B200_EINVAL, "workers (servers) must be in 1..33822 for CIMBA_B200_MODEL_HOLD (1..1080 with variant 1)");
        HoldArgs ha{};
        ha.workers = job->servers;
        ha.master_seed = job->master_seed;
        ha.first_trial = job->first_trial;
        ha.num_trials = job->num_trials;
        ha.duration = job->num_objects;
        ha.mean = job->arr_mean;
        ha.events = job->events;
        ha.objects = job->objects;
        ha.t_end = job->t_end;
        ha.sum_wait = job->sum_wait;
        ha.status = job->status;
        ha.max_queue = job->max_queue;
        ha.counters = job->counters;
        ha.trace_cap = job->trace_cap;
        ha.trace_key = job->trace_key;
        ha.trace_time = job->trace_time;
        if (!on_chip) {
            // hold_deep.cuh: levels >= 2 of the 32-ary heap in HBM/L2, persistent warps
            if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
                return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
            // variant 0 = the default below; 2 = one warp per trial (hold_deep.cuh); 3 / 4 = 16 / 8 lanes per trial
            const int lanes = job->variant == 2 ? 32 : (job->variant == 4 ? 8 : (job->variant == 3 ? 16 : HOLD_DEFAULT_LANES));
            const void *fn = lanes == 32 ? (trace ? (const void *)hold_deep_kernel<true> : (const void *)hold_deep_kernel<false>)
                           : lanes == 16 ? (trace ? (const void *)hold_group_kernel<16, true> : (const void *)hold_group_kernel<16, false>)
                                         : (trace ? (const void *)hold_group_kernel<8, true> : (const void *)hold_group_kernel<8, false>);
            int dev = 0, sms = 132, per_sm = 0;
            CUDA_TRY(cudaGetDevice(&dev));
            CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
            cudaError_t oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, DEEP_BLOCK, 0);
            if (oe != cudaSuccess || per_sm < 1) per_sm = 8;
            const uint64_t trials_per_block = (uint64_t)(DEEP_BLOCK / 32) * (uint64_t)(32 / lanes);
            const uint64_t resident = (uint64_t)sms * (uint64_t)per_sm;
            const uint64_t wanted = (job->num_trials + trials_per_block - 1) / trials_per_block;
            const unsigned blocks = (unsigned)(wanted < resident ? wanted : resident);
            DeepArgs da{};
            da.h = ha;
            da.rows = (uint4 *)job->workspace;
            da.row_entries = deep_row_entries(job->servers);
            void *kargs[] = { (void *)&da };
            cudaError_t le = cudaLaunchKernel(fn, dim3(blocks), dim3(DEEP_BLOCK), kargs, 0, st);
            g_launches++;
            cudaError_t e = le != cudaSuccess ? le : cudaGetLastError();
            return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "hold_deep_kernel launch");
        }
        // persistent one-warp CTAs: exactly as many as are resident at once (shared memory
        // bounds it at ~12 per SM), so no CTA waits for another to retire
        int dev = 0, sms = 132, per_sm = 0;
        CUDA_TRY(cudaGetDevice(&dev));
        CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        cudaError_t oe = trace
            ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hold_kernel<true>, 32, HOLD_SMEM_BYTES)
            : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, hold_kernel<false>, 32, HOLD_SMEM_BYTES);
        if (oe != cudaSuccess || per_sm < 1) per_sm = 8;
        const uint64_t resident = (uint64_t)sms * (uint64_t)per_sm;
        const unsigned blocks = (unsigned)(job->num_trials < resident ? job->num_trials : resident);
        if (trace) {
            hold_kernel<true><<<blocks, 32, HOLD_SMEM_BYTES, st>>>(ha);
        }
        else {
            hold_kernel<false><<<blocks, 32, HOLD_SMEM_BYTES, st>>>(ha);
        }
        g_launches++;
        cudaError_t e = cudaGetLastError();
        return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "hold_kernel launch");
    }
    return fail(CIMBA_B200_EINVAL, "unknown model");
}

namespace {
bool terrain_descriptor_ok(const cimba_b200_awacs_terrain *t)
{
    return t != nullptr && t->map != nullptr && t->cols >= 2u && t->rows >= 2u && t->x_scale > 0.0f && t->y_scale > 0.0f &&
           t->x_min < t->x_max && t->y_min < t->y_max && (uint64_t)t->cols * (uint64_t)t->rows <= 0xffffffffull;
}

// Registers `map` (a device pointer) for device `dev` and builds its tile-maximum map.  `owned` = the library made
// this copy (upload path) and frees it when it is replaced.  Caller holds no lock.
int register_terrain(int dev, const cimba_b200_awacs_terrain *t, const float *map, float *owned)
{
    const uint32_t tcols = (t->cols + AWACS_TILE - 1u) >> AWACS_TILE_SHIFT, trows = (t->rows + AWACS_TILE - 1u) >> AWACS_TILE_SHIFT;
    float *tiles = nullptr;
    CUDA_TRY(cudaMalloc(&tiles, (size_t)tcols * trows * sizeof(float)));
    aw_tile_max_kernel<<<dim3(tcols, trows), 256>>>(map, t->cols, t->rows, tiles, tcols);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        cudaFree(tiles);
        return cuda_fail(e, "aw_tile_max_kernel");
    }
    std::lock_guard<std::mutex> hold(g_terrain_mu);
    // no job may still be reading the previous registration (the caller's contract, as for any model input)
    if (g_terrain_tiles[dev] != nullptr) cudaFree(g_terrain_tiles[dev]);
    if (g_terrain_owned[dev] != nullptr && g_terrain_owned[dev] != owned) cudaFree(g_terrain_owned[dev]);
    g_terrain_tiles[dev] = tiles;
    g_terrain_owned[dev] = owned;
    g_terrain[dev] = AwacsTerrain{map, t->cols, t->rows, t->x_scale, t->y_scale, t->x_min, t->x_max, t->y_min, t->y_max,
                                  tiles, tcols, trows};
    g_terrain_set[dev] = true;
    return CIMBA_B200_OK;
}
}  // namespace

int cimba_b200_awacs_set_terrain(const cimba_b200_awacs_terrain *t)
{
    if (!terrain_descriptor_ok(t)) return fail(CIMBA_B200_EINVAL, "bad terrain descriptor (tutorial/tut_5_1.c:96-108)");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= MAX_TERRAIN_DEVICES) return fail(CIMBA_B200_EINVAL, "device index out of range");
    // a caller-owned map replaces (and frees) whatever copy an earlier upload left on this device
    return register_terrain(dev, t, t->map, nullptr);
}

int cimba_b200_awacs_upload_terrain(const cimba_b200_awacs_terrain *t)
{
    if (!terrain_descriptor_ok(t)) return fail(CIMBA_B200_EINVAL, "bad terrain descriptor (tutorial/tut_5_1.c:96-108)");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    if (dev < 0 || dev >= MAX_TERRAIN_DEVICES) return fail(CIMBA_B200_EINVAL, "device index out of range");
    const size_t bytes = (size_t)t->cols * (size_t)t->rows * sizeof(float);
    float *copy = nullptr;
    CUDA_TRY(cudaMalloc(&copy, bytes));
    cudaError_t e = cudaMemcpy(copy, t->map, bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(copy);
        return cuda_fail(e, "terrain upload");
    }
    const int rc = register_terrain(dev, t, copy, copy);
    if (rc != CIMBA_B200_OK) cudaFree(copy);
    return rc;
}

int cimba_b200_model_load(const char *path)
{
    if (path == nullptr) return fail(CIMBA_B200_EINVAL, "NULL path");
    void *h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
    if (h == nullptr) return fail(CIMBA_B200_EINVAL, "cannot load the model library: %s", dlerror());
    UserModel um{};
    um.handle = h;
    um.workspace_bytes = (uint64_t (*)(const cimba_b200_device_job *))dlsym(h, "cimba_b200_user_model_workspace_bytes");
    um.launch = (int (*)(const cimba_b200_device_job *, void *))dlsym(h, "cimba_b200_user_model_launch");
    const char *(*name)(void) = (const char *(*)(void))dlsym(h, "cimba_b200_user_model_name");
    if (um.workspace_bytes == nullptr || um.launch == nullptr || name == nullptr) {
        dlclose(h);
        return fail(CIMBA_B200_EINVAL, "%s does not export a model (end the model's .cu file with CMB_EXPORT_MODEL)", path);
    }
    um.name = name();
    std::lock_guard<std::mutex> hold(g_user_mu);
    g_user_models.push_back(um);
    return CIMBA_B200_MODEL_USER_BASE + (int)g_user_models.size() - 1;
}

const char *cimba_b200_model_name(int model_id)
{
    const UserModel *um = user_model(model_id);
    return um ? um->name.c_str() : nullptr;
}

int cimba_b200_summarize(const double *sum_wait, const uint64_t *objects,
                         uint64_t num_trials, double *out_summary, void *stream)
{
    if (sum_wait == nullptr || objects == nullptr || out_summary == nullptr || num_trials == 0u)
        return fail(CIMBA_B200_EINVAL, "bad argument to cimba_b200_summarize");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    summarize_kernel<<<1, SUMMARY_BLOCK, 0, (cudaStream_t)stream>>>(sum_wait, objects, num_trials, out_summary);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "summarize_kernel launch");
}

int cimba_b200_rng_draws(uint64_t seed, int kind, double p0, double p1,
                         uint64_t n, double *out, void *stream)
{
    if (out == nullptr || kind < 0 || kind > 8) return fail(CIMBA_B200_EINVAL, "bad argument to cimba_b200_rng_draws");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    rng_draws_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(seed, kind, p0, p1, n, out);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "rng_draws_kernel launch");
}

// cmb_random_alias_create, src/cmb_random.c:688-752 (Vose): host-side table construction;
// the tables are what rnd_alias_sample (csrc/distributions.cuh) reads on the device.
int cimba_b200_alias_create(uint32_t n, const double *pa, uint64_t *uprob, uint32_t *alias)
{
    if (n == 0u || pa == nullptr || uprob == nullptr || alias == nullptr)
        return fail(CIMBA_B200_EINVAL, "bad argument to cimba_b200_alias_create");
    std::vector<double> work(n);
    std::vector<uint32_t> small(n), large(n);
    double psum = 0.0;
    for (uint32_t i = 0; i < n; i++) {
        psum += pa[i];
        uprob[i] = 0u;
        alias[i] = 0u;
    }
    if (fabs(psum - 1.0) > 1.0e-3) return fail(CIMBA_B200_EINVAL, "probabilities must sum to one (src/cmb_random.c:634-642)");
    uint32_t ns = 0u, nl = 0u;
    for (uint32_t i = 0; i < n; i++) {
        work[i] = pa[i] * n / psum;
        if (work[i] < 1.0) small[ns++] = i;
        else large[nl++] = i;
    }
    while (ns > 0u && nl > 0u) {
        const uint32_t l = small[--ns];
        const uint32_t g = large[--nl];
        uprob[l] = alias_secure(work[l]);
        alias[l] = g;
        work[g] = (work[g] + work[l]) - 1.0;
        if (work[g] < 1.0) small[ns++] = g;
        else large[nl++] = g;
    }
    while (nl > 0u) uprob[large[--nl]] = UINT64_MAX;
    while (ns > 0u) uprob[small[--ns]] = UINT64_MAX;
    return CIMBA_B200_OK;
}

int cimba_b200_rng_draws_ex(uint64_t seed, int kind, const double *params, uint32_t num_params,
                            uint64_t n, double *out, void *stream)
{
    if (out == nullptr || kind < 9 || kind > 33 || num_params > CIMBA_B200_RNG_MAX_PARAMS ||
        (num_params > 0u && params == nullptr))
        return fail(CIMBA_B200_EINVAL, "bad argument to cimba_b200_rng_draws_ex");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    DrawParams par{};
    for (uint32_t i = 0; i < num_params; i++) par.v[i] = params[i];
    // kinds that carry an array inline: {n, v[n]} (13 hypoexponential, 29 loaded dice, 30 alias), {n, m[n], p[n]} (14
    // hyperexponential); 26 / 27 / 33 read {n, p}.  The kernel indexes par.v[] by n: refuse what does not fit.
    if (kind == 13 || kind == 14 || kind == 29 || kind == 30 || kind == 26 || kind == 27 || kind == 33) {
        const double n = num_params > 0u ? params[0] : 0.0;
        if (!(n >= 1.0) || !(n <= 4294967295.0) || n != floor(n))
            return fail(CIMBA_B200_EINVAL, "params[0] must be a count >= 1 for this distribution");
        const uint64_t cnt = (uint64_t)n;
        const uint64_t need = (kind == 14) ? 1u + 2u * cnt : ((kind == 26 || kind == 27 || kind == 33) ? 2u : 1u + cnt);
        if (need > num_params) return fail(CIMBA_B200_EINVAL, "params: the count in params[0] does not fit num_params");
    }
    if (kind == 30) {
        const uint32_t cnt = num_params > 0u ? (uint32_t)params[0] : 0u;
        if (cnt == 0u || cnt + 1u > num_params) return fail(CIMBA_B200_EINVAL, "alias: params = {n, p[0..n-1]}");
        const int rc = cimba_b200_alias_create(cnt, params + 1, par.uprob, par.alias);
        if (rc != CIMBA_B200_OK) return rc;
    }
    rng_draws_ex_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(seed, kind, par, n, out);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "rng_draws_ex_kernel launch");
}

// ------------------------------------------------------------ host-buffer path

namespace {
constexpr int MAX_CACHED_DEVICES = 64;

struct DeviceCache {           // per-device staging + arena + stream of the host-buffer path
    std::mutex   mu;
    void        *dev = nullptr, *h_in = nullptr, *h_out = nullptr;
    size_t       dev_bytes = 0, h_in_bytes = 0, h_out_bytes = 0;
    cudaStream_t st = nullptr;

    int reserve_host(size_t in_bytes, size_t out_bytes)
    {
        if (in_bytes > h_in_bytes) {
            if (h_in) cudaFreeHost(h_in);
            h_in = nullptr;
            h_in_bytes = 0;
            CUDA_TRY(cudaMallocHost(&h_in, in_bytes));
            h_in_bytes = in_bytes;
        }
        if (out_bytes > h_out_bytes) {
            if (h_out) cudaFreeHost(h_out);
            h_out = nullptr;
            h_out_bytes = 0;
            CUDA_TRY(cudaMallocHost(&h_out, out_bytes));
            h_out_bytes = out_bytes;
        }
        return CIMBA_B200_OK;
    }
    int reserve_device(size_t bytes)
    {
        if (st == nullptr) CUDA_TRY(cudaStreamCreate(&st));
        if (bytes > dev_bytes) {
            if (dev) cudaFree(dev);
            dev = nullptr;
            dev_bytes = 0;
            CUDA_TRY(cudaMalloc(&dev, bytes));
            dev_bytes = bytes;
        }
        return CIMBA_B200_OK;
    }
    void release()
    {
        if (dev) cudaFree(dev);
        if (h_in) cudaFreeHost(h_in);
        if (h_out) cudaFreeHost(h_out);
        if (st) cudaStreamDestroy(st);
        dev = h_in = h_out = nullptr;
        dev_bytes = h_in_bytes = h_out_bytes = 0;
        st = nullptr;
    }
};
DeviceCache g_cache[MAX_CACHED_DEVICES];

struct PhaseClock {            // CIMBA_B200_TIMING=1: phase times of the host-buffer path on stderr
    bool on;
    std::chrono::steady_clock::time_point t;
    PhaseClock() : on(getenv("CIMBA_B200_TIMING") != nullptr), t(std::chrono::steady_clock::now()) {}
    void lap(const char *what)
    {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[cimba_b200] %-28s %9.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t).count());
        t = now;
    }
};
}  // namespace

namespace {
int run_experiment_chunk(void *array, uint64_t num_trials, size_t stride, const cimba_b200_experiment *d);

// Trials per launch of the host-buffer path.  An experiment larger than this runs as consecutive chunks
// (seeds depend on the global trial index only), so staging and workspace stay bounded - 1 Mi M/M/1
// trials need 4.3 GB of spill ring - while every chunk still saturates the GPU (M/M/1 peaks at ~6e5).
uint64_t chunk_trials()
{
    const char *env = getenv("CIMBA_B200_CHUNK_TRIALS");
    if (env != nullptr) {
        const unsigned long long v = strtoull(env, nullptr, 10);
        if (v > 0ull) return (uint64_t)v;
    }
    return 1ull << 20;
}
}  // namespace

int cimba_b200_run_experiment(void *array, uint64_t num_trials, size_t stride,
                              const cimba_b200_experiment *d)
{
    if (array == nullptr || d == nullptr) return fail(CIMBA_B200_EINVAL, "NULL experiment array or descriptor");
    if (num_trials == 0u || stride == 0u) return fail(CIMBA_B200_EINVAL, "num_trials and trial_struct_size must be > 0");
    const uint64_t chunk = chunk_trials();
    int worst = CIMBA_B200_OK;
    for (uint64_t off = 0; off < num_trials; off += chunk) {
        const uint64_t m = num_trials - off < chunk ? num_trials - off : chunk;
        cimba_b200_experiment sub = *d;
        sub.first_trial = d->first_trial + off;
        const int rc = run_experiment_chunk((char *)array + off * stride, m, stride, &sub);
        if (rc == CIMBA_B200_ETRIAL) {
            worst = rc;                                 // the other trials' results are valid: carry on
        }
        else if (rc != CIMBA_B200_OK) {
            return rc;
        }
    }
    if (worst != CIMBA_B200_OK) return fail(worst, "at least one trial reported a capacity violation");
    return CIMBA_B200_OK;
}

namespace {
int run_experiment_chunk(void *array, uint64_t num_trials, size_t stride, const cimba_b200_experiment *d)
{
    PhaseClock clk;
    if (array == nullptr || d == nullptr) return fail(CIMBA_B200_EINVAL, "NULL experiment array or descriptor");
    if (num_trials == 0u || stride == 0u) return fail(CIMBA_B200_EINVAL, "num_trials and trial_struct_size must be > 0");
    if (d->model == CIMBA_B200_MODEL_AWACS)
        return fail(CIMBA_B200_EINVAL, "MODEL_AWACS runs through the device-resident interface (its terrain lives in HBM)");
    if (d->off_arr_mean == CIMBA_B200_NO_FIELD || d->off_srv_mean == CIMBA_B200_NO_FIELD)
        return fail(CIMBA_B200_EINVAL, "off_arr_mean and off_srv_mean are required");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    // the caller's current device is the caller's: put it back on every way out
    struct DeviceGuard {
        int before = -1;
        bool armed = false;
        ~DeviceGuard() { if (armed) (void)cudaSetDevice(before); }
    } restore;
    if (d->device >= 0) {
        CUDA_TRY(cudaGetDevice(&restore.before));
        CUDA_TRY(cudaSetDevice(d->device));
        restore.armed = restore.before != d->device;
    }

    const uint64_t n = num_trials;
    char *base = (char *)array;

    // gather the two input columns into pinned staging, scatter results back the same way.
    // Staging, the device arena and the stream are kept per device between calls (grow-only):
    // cudaMallocHost / cudaMalloc / cudaFree of the ~270 MB a 65 536-trial job needs would
    // otherwise be paid on every call.
    int devno = 0;
    CUDA_TRY(cudaGetDevice(&devno));
    if (devno < 0 || devno >= MAX_CACHED_DEVICES) return fail(CIMBA_B200_EINVAL, "device index out of range");
    DeviceCache &cache = g_cache[devno];
    std::lock_guard<std::mutex> hold(cache.mu);
    // counters (8 words per trial) travel only when the caller asks for them; the device side always has
    // them because some models write nothing else of interest
    const bool want_counters = d->off_counters != CIMBA_B200_NO_FIELD;
    const size_t out_row = 2 * sizeof(uint64_t) + 2 * sizeof(double) + sizeof(uint32_t) + sizeof(uint32_t);
    const size_t cnt_row = 8 * sizeof(uint64_t);
    {
        const int rc0 = cache.reserve_host(2 * n * sizeof(double), n * (out_row + (want_counters ? cnt_row : 0)));
        if (rc0 != CIMBA_B200_OK) return rc0;
    }
    double *h_in = (double *)cache.h_in;
    unsigned char *h_out = (unsigned char *)cache.h_out;
    clk.lap("pinned staging alloc");
    for (uint64_t i = 0; i < n; i++) {
        memcpy(&h_in[i], base + i * stride + d->off_arr_mean, sizeof(double));
        memcpy(&h_in[n + i], base + i * stride + d->off_srv_mean, sizeof(double));
    }
    clk.lap("gather inputs");

    cimba_b200_device_job job{};
    job.model = d->model;
    job.servers = d->servers;
    job.mapping = d->mapping;
    job.variant = d->variant;
    job.queue_spill_cap = d->queue_spill_cap;
    job.params = d->params;
    job.num_params = d->num_params;
    job.master_seed = d->master_seed;
    job.first_trial = d->first_trial;
    job.num_trials = n;
    job.num_objects = d->num_objects;

    unsigned char *dev = nullptr;
    const uint64_t ws = cimba_b200_workspace_bytes(&job);
    const size_t in_bytes = 2 * n * sizeof(double);
    const size_t out_bytes = n * out_row;
    const size_t cnt_bytes = n * cnt_row;
    int rc = cache.reserve_device(in_bytes + out_bytes + cnt_bytes + ws + 256);
    if (rc != CIMBA_B200_OK) return rc;
    dev = (unsigned char *)cache.dev;
    cudaStream_t st = cache.st;
    cudaError_t e = cudaSuccess;
    clk.lap("stream + device alloc");
    {
        double *d_in = (double *)dev;
        unsigned char *d_out = dev + in_bytes;
        job.arr_mean = d_in;
        job.srv_mean = d_in + n;
        job.events = (uint64_t *)d_out;
        job.objects = job.events + n;
        job.t_end = (double *)(job.objects + n);
        job.sum_wait = job.t_end + n;
        job.status = (uint32_t *)(job.sum_wait + n);
        job.max_queue = job.status + n;
        job.counters = (uint64_t *)(d_out + out_bytes);
        job.workspace = dev + ((in_bytes + out_bytes + cnt_bytes + 255) / 256) * 256;
        job.workspace_bytes = ws;

        e = cudaMemcpyAsync(d_in, h_in, in_bytes, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) { rc = cuda_fail(e, "H2D"); goto done; }
        // the arena is reused between calls and many kernels (M/M/1, M/M/c, ...) write no counters: without this the
        // caller's counters field would receive whatever an earlier call left at these addresses
        if (want_counters) {
            e = cudaMemsetAsync(job.counters, 0, cnt_bytes, st);
            if (e != cudaSuccess) { rc = cuda_fail(e, "counters memset"); goto done; }
        }
        rc = cimba_b200_launch(&job, st);
        if (rc != CIMBA_B200_OK) goto done;
        e = cudaMemcpyAsync(h_out, d_out, out_bytes + (want_counters ? cnt_bytes : 0), cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) { rc = cuda_fail(e, "D2H"); goto done; }
        e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { rc = cuda_fail(e, "cudaStreamSynchronize"); goto done; }
        clk.lap("H2D + kernel + D2H");

        const uint64_t *ev = (const uint64_t *)h_out;
        const uint64_t *ob = ev + n;
        const double *te = (const double *)(ob + n);
        const double *sw = te + n;
        const uint32_t *stt = (const uint32_t *)(sw + n);
        const uint32_t *mq = stt + n;
        const uint64_t *cnt = (const uint64_t *)(h_out + out_bytes);
        bool any_bad = false;
        for (uint64_t i = 0; i < n; i++) {
            char *row = base + i * stride;
            if (d->off_obj_cnt != CIMBA_B200_NO_FIELD) memcpy(row + d->off_obj_cnt, &ob[i], 8);
            if (d->off_sum_wait != CIMBA_B200_NO_FIELD) memcpy(row + d->off_sum_wait, &sw[i], 8);
            if (d->off_avg_wait != CIMBA_B200_NO_FIELD) {
                const double avg = sw[i] / (double)ob[i];
                memcpy(row + d->off_avg_wait, &avg, 8);
            }
            if (d->off_events != CIMBA_B200_NO_FIELD) memcpy(row + d->off_events, &ev[i], 8);
            if (d->off_t_end != CIMBA_B200_NO_FIELD) memcpy(row + d->off_t_end, &te[i], 8);
            if (d->off_status != CIMBA_B200_NO_FIELD) memcpy(row + d->off_status, &stt[i], 4);
            if (d->off_max_queue != CIMBA_B200_NO_FIELD) memcpy(row + d->off_max_queue, &mq[i], 4);
            if (want_counters) memcpy(row + d->off_counters, &cnt[i * 8u], cnt_row);
            any_bad |= (stt[i] != 0u);
        }
        if (any_bad) rc = fail(CIMBA_B200_ETRIAL, "at least one trial reported a capacity violation");
        clk.lap("scatter results");
    }
done:
    return rc;
}
}  // namespace

void cimba_b200_release_cache(void)
{
    int count = cimba_b200_device_count();
    if (count > MAX_CACHED_DEVICES) count = MAX_CACHED_DEVICES;
    int before = 0;
    if (count > 0) cudaGetDevice(&before);
    for (int g = 0; g < count; g++) {
        std::lock_guard<std::mutex> hold(g_cache[g].mu);
        if (g_cache[g].dev || g_cache[g].h_in || g_cache[g].h_out || g_cache[g].st) {
            cudaSetDevice(g);
            g_cache[g].release();
        }
    }
    {
        std::lock_guard<std::mutex> hold(g_terrain_mu);
        for (int g = 0; g < count && g < MAX_TERRAIN_DEVICES; g++) {
            if (g_terrain_owned[g] != nullptr) {
                // the registered map IS the library's copy (register_terrain frees a stale copy when a caller-owned
                // map replaces it), so the registration goes with it; a caller-owned registration stays valid
                cudaSetDevice(g);
                cudaFree(g_terrain_owned[g]);
                g_terrain_owned[g] = nullptr;
                if (g_terrain_tiles[g] != nullptr) cudaFree(g_terrain_tiles[g]);
                g_terrain_tiles[g] = nullptr;
                g_terrain_set[g] = false;
            }
        }
    }
    if (count > 0) cudaSetDevice(before);
}

namespace {
std::mutex g_hook_mu;
cimba_b200_thread_init_func *g_hook_init = nullptr;
cimba_b200_thread_exit_func *g_hook_exit = nullptr;
void *g_hook_usrarg = nullptr;
thread_local void *t_thread_context = nullptr;
}  // namespace

void cimba_b200_set_thread_hooks(cimba_b200_thread_init_func *initfunc, void *usrarg, cimba_b200_thread_exit_func *exitfunc)
{   // src/cimba.c:65-73
    std::lock_guard<std::mutex> hold(g_hook_mu);
    g_hook_init = initfunc;
    g_hook_usrarg = usrarg;
    g_hook_exit = exitfunc;
}

void *cimba_b200_thread_context(void) { return t_thread_context; }     // src/cimba.c:75-78

// The reference's executive starts one pthread per logical core and lets them pull
// trials (src/cimba.c:151-188).  The counterpart here: one host thread per GPU, each
// running a contiguous block of the trial array on its own device and stream.  Seeds
// depend on the global trial index only, so results do not depend on the GPU count.
int cimba_b200_run_experiment_all_gpus(void *array, uint64_t num_trials, size_t stride,
                                       const cimba_b200_experiment *d, int max_gpus)
{
    if (array == nullptr || d == nullptr) return fail(CIMBA_B200_EINVAL, "NULL experiment array or descriptor");
    if (num_trials == 0u || stride == 0u) return fail(CIMBA_B200_EINVAL, "num_trials and trial_struct_size must be > 0");
    int gpus = cimba_b200_device_count();
    if (gpus <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    if (max_gpus > 0 && max_gpus < gpus) gpus = max_gpus;
    if ((uint64_t)gpus > num_trials) gpus = (int)num_trials;

    std::vector<int> rc((size_t)gpus, CIMBA_B200_OK);
    std::vector<std::string> msg((size_t)gpus);
    std::vector<std::thread> pool;
    for (int g = 0; g < gpus; g++) {
        pool.emplace_back([&, g]() {
            const uint64_t lo = num_trials * (uint64_t)g / (uint64_t)gpus;
            const uint64_t hi = num_trials * (uint64_t)(g + 1) / (uint64_t)gpus;
            cimba_b200_experiment mine = *d;
            mine.device = g;
            mine.first_trial = d->first_trial + lo;
            cimba_b200_thread_init_func *init;
            cimba_b200_thread_exit_func *done;
            void *usrarg;
            {
                std::lock_guard<std::mutex> hold(g_hook_mu);
                init = g_hook_init;
                done = g_hook_exit;
                usrarg = g_hook_usrarg;
            }
            (void)cudaSetDevice(g);
            if (init != nullptr) t_thread_context = init(usrarg, (uint64_t)g);      // src/cimba.c:102-104
            rc[(size_t)g] = cimba_b200_run_experiment((char *)array + lo * stride, hi - lo, stride, &mine);
            msg[(size_t)g] = g_err;                     // thread-local message of this worker
            if (done != nullptr) done(t_thread_context);                            // thread_exit_wrapper, :80-86
            t_thread_context = nullptr;
        });
    }
    for (auto &t : pool) {
        t.join();
    }
    int worst = CIMBA_B200_OK;
    for (int g = 0; g < gpus; g++) {
        if (rc[(size_t)g] != CIMBA_B200_OK && (worst == CIMBA_B200_OK || worst == CIMBA_B200_ETRIAL)) {
            worst = rc[(size_t)g];
            snprintf(g_err, sizeof(g_err), "GPU %d: %s", g, msg[(size_t)g].c_str());
        }
    }
    return worst;
}

int cimba_b200_summarize_weighted(const double *x, const double *w, uint64_t n,
                                  uint64_t *out_row, void *stream)
{
    if (x == nullptr || w == nullptr || out_row == nullptr || n == 0u)
        return fail(CIMBA_B200_EINVAL, "bad argument to cimba_b200_summarize_weighted");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    summarize_weighted_kernel<<<1, SUMMARY_BLOCK, 0, (cudaStream_t)stream>>>(x, w, n, out_row);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "summarize_weighted_kernel launch");
}

int cimba_b200_merge_weighted_rows(const uint64_t *rows, uint64_t n, uint64_t *out_row, void *stream)
{
    if (rows == nullptr || out_row == nullptr || n == 0u)
        return fail(CIMBA_B200_EINVAL, "bad argument to cimba_b200_merge_weighted_rows");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    merge_weighted_rows_kernel<<<1, SUMMARY_BLOCK, 0, (cudaStream_t)stream>>>(rows, n, out_row);
    g_launches++;
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, "merge_weighted_rows_kernel launch");
}

// ------------------------------------------------- cmb_wtdsummary on the host
namespace {
WtdAcc wtd_from(const cimba_b200_wtdsummary *s)
{
    return WtdAcc{s->base.count, s->base.min, s->base.max, s->base.m1, s->base.m2, s->base.m3, s->base.m4, s->wsum};
}
void wtd_to(const WtdAcc &a, cimba_b200_wtdsummary *s)
{
    cimba_b200_datasummary_initialize(&s->base);
    s->base.count = a.count;
    s->base.min = a.min;
    s->base.max = a.max;
    s->base.m1 = a.m1;
    s->base.m2 = a.m2;
    s->base.m3 = a.m3;
    s->base.m4 = a.m4;
    s->wsum = a.wsum;
}
}  // namespace

void cimba_b200_wtdsummary_initialize(cimba_b200_wtdsummary *s)
{   // src/cmb_wtdsummary.c:40-46
    cimba_b200_datasummary_initialize(&s->base);
    s->wsum = 0.0;
}

uint64_t cimba_b200_wtdsummary_add(cimba_b200_wtdsummary *s, double x, double w)
{
    WtdAcc a = wtd_from(s);
    wtd_add(a, x, w);
    wtd_to(a, s);
    return s->base.count;
}

uint64_t cimba_b200_wtdsummary_merge(cimba_b200_wtdsummary *tgt, const cimba_b200_wtdsummary *p,
                                     const cimba_b200_wtdsummary *q)
{
    const WtdAcc c = wtd_merge(wtd_from(p), wtd_from(q));
    wtd_to(c, tgt);
    return tgt->base.count;
}

double cimba_b200_wtdsummary_mean(const cimba_b200_wtdsummary *s) { return s->base.m1; }

double cimba_b200_wtdsummary_variance(const cimba_b200_wtdsummary *s)
{   // include/cmb_wtdsummary.h:192-197 delegates to cmb_datasummary_variance on the base part
    return cimba_b200_datasummary_variance(&s->base);
}

// ------------------------------------------------- cmb_datasummary on the host

void cimba_b200_datasummary_initialize(cimba_b200_datasummary *s)
{   // src/cmb_datasummary.c:37-50
    s->cookie = 0x1ce1ce1ce1ce1ce1ull;
    s->count = 0u;
    s->min = DBL_MAX;
    s->max = -DBL_MAX;
    s->m1 = s->m2 = s->m3 = s->m4 = 0.0;
}

uint64_t cimba_b200_datasummary_add(cimba_b200_datasummary *s, double y)
{
    SummaryAcc a{s->count, s->min, s->max, s->m1, s->m2, s->m3, s->m4};
    summary_add(a, y);
    s->count = a.count; s->min = a.min; s->max = a.max;
    s->m1 = a.m1; s->m2 = a.m2; s->m3 = a.m3; s->m4 = a.m4;
    return s->count;
}

uint64_t cimba_b200_datasummary_merge(cimba_b200_datasummary *tgt,
                                      const cimba_b200_datasummary *p,
                                      const cimba_b200_datasummary *q)
{
    const SummaryAcc a{p->count, p->min, p->max, p->m1, p->m2, p->m3, p->m4};
    const SummaryAcc b{q->count, q->min, q->max, q->m1, q->m2, q->m3, q->m4};
    const SummaryAcc c = summary_merge(a, b);
    cimba_b200_datasummary_initialize(tgt);
    tgt->count = c.count; tgt->min = c.min; tgt->max = c.max;
    tgt->m1 = c.m1; tgt->m2 = c.m2; tgt->m3 = c.m3; tgt->m4 = c.m4;
    return tgt->count;
}

double cimba_b200_datasummary_mean(const cimba_b200_datasummary *s) { return s->m1; }

double cimba_b200_datasummary_variance(const cimba_b200_datasummary *s)
{   // include/cmb_datasummary.h:197-210 (sample variance)
    return (s->count > 1u) ? s->m2 / (double)(s->count - 1u) : 0.0;
}

double cimba_b200_datasummary_stddev(const cimba_b200_datasummary *s)
{
    return sqrt(cimba_b200_datasummary_variance(s));
}

uint64_t cimba_b200_datasummary_count(const cimba_b200_datasummary *s) { return s->count; }
double cimba_b200_datasummary_max(const cimba_b200_datasummary *s) { return s->max; }
double cimba_b200_datasummary_min(const cimba_b200_datasummary *s) { return s->min; }

double cimba_b200_datasummary_skewness(const cimba_b200_datasummary *s)
{   // src/cmb_datasummary.c:214-230: population estimate, then the finite-sample correction
    if (s->count <= 2u) return 0.0;
    const double n = (double)s->count;
    const double g = sqrt(n) * s->m3 / pow(s->m2, 1.5);
    return sqrt(n * (n - 1.0)) * g / (n - 2.0);
}

double cimba_b200_datasummary_kurtosis(const cimba_b200_datasummary *s)
{   // src/cmb_datasummary.c:233-249: sample excess kurtosis
    if (s->count <= 3u) return 0.0;
    const double n = (double)s->count;
    const double g = n * s->m4 / (s->m2 * s->m2) - 3.0;
    return (n - 1.0) / ((n - 2.0) * (n - 3.0)) * ((n + 1.0) * g + 6.0);
}

void cimba_b200_datasummary_print(const cimba_b200_datasummary *s, FILE *fp, int lead_ins)
{   // src/cmb_datasummary.c:168-212: one line, a column only when the count supports the statistic
    if (s == nullptr || fp == nullptr) return;
    const bool li = lead_ins != 0;
    fprintf(fp, "%s%8llu", li ? "N " : "", (unsigned long long)s->count);
    if (s->count > 0u) fprintf(fp, "%s%#8.4g", li ? "  Mean " : "\t", cimba_b200_datasummary_mean(s));
    if (s->count > 1u) {
        const double var = cimba_b200_datasummary_variance(s);
        fprintf(fp, "%s%#8.4g", li ? "  StdDev " : "\t", sqrt(var));
        fprintf(fp, "%s%#8.4g", li ? "  Variance " : "\t", var);
    }
    if (s->count > 2u) fprintf(fp, "%s%#8.4g", li ? "  Skewness " : "\t", cimba_b200_datasummary_skewness(s));
    if (s->count > 3u) fprintf(fp, "%s%#8.4g", li ? "  Kurtosis " : "\t", cimba_b200_datasummary_kurtosis(s));
    fprintf(fp, "\n");
}

double cimba_b200_wtdsummary_stddev(const cimba_b200_wtdsummary *s) { return cimba_b200_datasummary_stddev(&s->base); }
double cimba_b200_wtdsummary_skewness(const cimba_b200_wtdsummary *s) { return cimba_b200_datasummary_skewness(&s->base); }
double cimba_b200_wtdsummary_kurtosis(const cimba_b200_wtdsummary *s) { return cimba_b200_datasummary_kurtosis(&s->base); }
void cimba_b200_wtdsummary_print(const cimba_b200_wtdsummary *s, FILE *fp, int lead_ins)
{
    if (s != nullptr) cimba_b200_datasummary_print(&s->base, fp, lead_ins);
}

}  // extern "C"
