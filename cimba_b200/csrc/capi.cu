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

// growth arena of the repair pass behind the fixed-capacity kernels of the library (M/M/1, G/G/1, M/M/c, models 3-6, 8, 11-14)
uint64_t repair_arena_bytes(const cimba_b200_device_job *job)
{
    uint64_t b = job->num_trials * 32768ull;
    if (b < (64ull << 20)) b = 64ull << 20;
    if (b > (4ull << 30)) b = 4ull << 30;
    return cmb::ARENA_HEADER + b;
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

// ---------------------------------------------------------------- routes
// A route is the code that serves a job: what workspace it needs and how it launches.  route() picks it; its launch
// runs after cimba_b200_launch's common checks and makes the checks of its own.
struct Route {
    uint64_t (*workspace)(const cimba_b200_device_job *);
    int (*launch)(const cimba_b200_device_job *, cudaStream_t);
};

int mapping_of(const cimba_b200_device_job *job) { return job->mapping == 0 ? CIMBA_B200_MAP_LANE : job->mapping; }

int check_workspace(const cimba_b200_device_job *job)
{
    if (job->workspace_bytes < cimba_b200_workspace_bytes(job) || job->workspace == nullptr)
        return fail(CIMBA_B200_EINVAL, "workspace too small; see cimba_b200_workspace_bytes()");
    return CIMBA_B200_OK;
}

// a launch made by cmb_launch.cuh (a cudaError_t as int) that started `launches` kernels
int counted(int e, const char *what, int launches = 1)
{
    g_launches += launches;
    return e == 0 ? CIMBA_B200_OK : cuda_fail((cudaError_t)e, what);
}

// a kernel of the library, in its TRACE instantiation when the job records pops
template <class Args>
int launch_kernel(const cimba_b200_device_job *job, void (*plain)(Args), void (*traced)(Args), dim3 grid, unsigned block,
                  size_t smem, cudaStream_t st, const Args &a, const char *what)
{
    void (*const kernel)(Args) = job->trace_cap > 0u ? traced : plain;
    kernel<<<grid, block, smem, st>>>(a);
    g_launches++;
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? CIMBA_B200_OK : cuda_fail(e, what);
}

// after a fixed-capacity kernel (result e): the general engine re-runs what it flagged, in all of the workspace behind its
// rings - so a caller whose trials come back CIMBA_B200_TRIAL_ARENA_EXHAUSTED cures that with a larger workspace
template <class Model>
int then_repair(int e, const cimba_b200_device_job *job, uint64_t rings_bytes, cudaStream_t st, const char *what)
{
    if (e != CIMBA_B200_OK || job->status == nullptr) return e;       // nobody could see a flag: nothing to repair by
    return counted(cmb::launch_repair<Model>(*job, rings_bytes, job->workspace_bytes - cmb::align256(rings_bytes), st), what);
}

// persistent CTAs: as many as are resident at once (`fallback` per SM if the occupancy query fails), at most `wanted`
int resident_grid(const void *fn, int block, size_t smem, int fallback, uint64_t wanted, unsigned *grid)
{
    int dev = 0, sms = 132, per_sm = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    cudaError_t oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, block, smem);
    if (oe != cudaSuccess || per_sm < 1) per_sm = fallback;
    const uint64_t resident = (uint64_t)sms * (uint64_t)per_sm;
    *grid = (unsigned)(wanted < resident ? wanted : resident);
    return CIMBA_B200_OK;
}

// ---- the general engine over every trial (growable event list, wait lists and queues)
template <class Model>
uint64_t engine_workspace(const cimba_b200_device_job *job) { return cmb::workspace_bytes_for<Model>(*job); }

// servers_msg = NULL: the model has no capacity to check
int engine_checks(const cimba_b200_device_job *job, const char *servers_msg)
{
    if (mapping_of(job) != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "the general engine runs one trial per lane (CIMBA_B200_MAP_LANE)");
    if (servers_msg != nullptr && job->servers < 1) return fail(CIMBA_B200_EINVAL, servers_msg);
    return check_workspace(job);
}

template <class Model>
int launch_engine(const cimba_b200_device_job *job, cudaStream_t st, const char *what)
{
    return counted(cmb::launch_model<Model>(*job, (unsigned char *)job->workspace, job->workspace_bytes, 0u, st), what);
}

template <class Model> const char *const ENGINE_WHAT = nullptr;
template <> const char *const ENGINE_WHAT<models::MM1> = "trial_kernel<MM1> launch";
template <> const char *const ENGINE_WHAT<models::GG1> = "trial_kernel<GG1> launch";
template <> const char *const ENGINE_WHAT<models::MM1Recorded> = "trial_kernel<MM1Recorded> launch";
template <> const char *const ENGINE_WHAT<models::MMC> = "trial_kernel<MMC> launch";
template <> const char *const ENGINE_WHAT<models::HoldGeneral> = "trial_kernel<HoldGeneral> launch";
template <> const char *const ENGINE_WHAT<models::Renege> = "trial_kernel<Renege> launch";
template <> const char *const ENGINE_WHAT<models::Cheese> = "trial_kernel<Cheese> launch";
template <> const char *const ENGINE_WHAT<models::Tutorial1> = "trial_kernel<Tutorial1> launch";
template <> const char *const ENGINE_WHAT<models::Park> = "trial_kernel<Park> launch";
template <> const char *const ENGINE_WHAT<models::Tutorial2> = "trial_kernel<Tutorial2> launch";

template <class Model>
int engine_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (const int e = engine_checks(job, "servers must be >= 1")) return e;
    return launch_engine<Model>(job, st, ENGINE_WHAT<Model>);
}

template <class Model>
constexpr Route ENGINE{engine_workspace<Model>, engine_launch<Model>};

int harbor_engine_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (const int e = engine_checks(job, "servers must be >= 1")) return e;
    if (job->servers < 3) return fail(CIMBA_B200_EINVAL, "tugs (servers) must be >= 3 for CIMBA_B200_MODEL_HARBOR (a large ship needs 3)");
    return launch_engine<models::HarborGeneral>(job, st, "trial_kernel<HarborGeneral> launch");
}

// ---- the static tier (cmb_static.cuh): ModelT<StaticSim<NPROC, NQUEUE>> first, ModelT<Sim> for what it flags
template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT = 0>
uint64_t static_workspace(const cimba_b200_device_job *job) { return cmb::workspace_bytes_static<ModelT, NPROC, NQUEUE, NEVENT>(*job); }

template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT = 0>
int static_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (mapping_of(job) != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "the static tier runs one trial per lane (CIMBA_B200_MAP_LANE)");
    if (const int e = check_workspace(job)) return e;
    return counted(cmb::launch_static_model<ModelT, NPROC, NQUEUE, NEVENT>(*job, st), "static_trial_kernel launch",
                   job->status != nullptr ? 2 : 1);
}

template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT = 0>
constexpr Route STATIC{static_workspace<ModelT, NPROC, NQUEUE, NEVENT>, static_launch<ModelT, NPROC, NQUEUE, NEVENT>};

// ... for a model without queues whose other routes already size its jobs (models 14, 18, 21): the tier keeps no rings, and its
// repair pass grows the general engine's containers in the workspace WORKSPACE asks for - so a job needs the same workspace
// whichever variant serves it.  SERVERS: refuse servers < 1, as the model's general-engine route does.
template <template <class> class ModelT, int NPROC, int NEVENT, uint64_t (*WORKSPACE)(const cimba_b200_device_job *), bool SERVERS>
int static_launch_in(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (mapping_of(job) != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "the static tier runs one trial per lane (CIMBA_B200_MAP_LANE)");
    if (SERVERS && job->servers < 1) return fail(CIMBA_B200_EINVAL, "servers must be >= 1");
    if (const int e = check_workspace(job)) return e;
    return counted(cmb::launch_static_trials<ModelT, NPROC, 0, NEVENT>(*job, st), "static_trial_kernel launch",
                   job->status != nullptr ? 2 : 1);
}

template <template <class> class ModelT, int NPROC, int NEVENT, uint64_t (*WORKSPACE)(const cimba_b200_device_job *), bool SERVERS>
constexpr Route STATIC_IN{WORKSPACE, static_launch_in<ModelT, NPROC, NEVENT, WORKSPACE, SERVERS>};

// ---- the fused M/M/1, G/G/1 and M/M/c kernels: a queue window on chip, a ring per trial in HBM
uint64_t queue_rings_bytes(const cimba_b200_device_job *job)
{
    const uint32_t cap = cmb::spill_cap(*job);
    return job->num_trials * (uint64_t)(cap == 0u ? cmb::SPILL_CAP_DEFAULT : cap) * sizeof(double);
}

uint64_t queue_workspace(const cimba_b200_device_job *job) { return cmb::rings_then_arena(queue_rings_bytes(job), repair_arena_bytes(job)); }

// 8 CTAs of mm1_kernel per SM (65 536 trials in one wave on 132 SMs) need 8 x (27 136 + 1 024) B = 220 KB of shared memory,
// which only the largest carveout gives; with a smaller split the driver might pick, the launch would take two waves.  Both
// instantiations ask for it, once per device (about 28 KB of the SM's unified L1 / shared memory stay L1).
int mm1_prefer_shared()
{
    static std::atomic<uint64_t> done{0};           // one bit per device
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    const uint64_t bit = dev < 64 ? 1ull << dev : 0ull;
    if (bit != 0u && (done.load() & bit) != 0u) return CIMBA_B200_OK;
    CUDA_TRY(cudaFuncSetAttribute(mm1_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CUDA_TRY(cudaFuncSetAttribute(mm1_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    done.fetch_or(bit);
    return CIMBA_B200_OK;
}

int queue_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (const int e = check_workspace(job)) return e;
    const int mapping = mapping_of(job);
    QueueArgs qa = cmb::job_args<QueueArgs>(*job);
    qa.mapping = mapping;
    qa.num_objects = job->num_objects;
    qa.arr_mean = job->arr_mean;
    qa.srv_mean = job->srv_mean;
    qa.counters = job->counters;
    qa.spill = (double *)job->workspace;
    qa.spill_cap = cmb::spill_cap(*job);
    qa.diag = (unsigned long long *)job->diag;
    const uint64_t threads = job->num_trials * (uint64_t)mapping;
    const uint64_t blocks = (threads + QUEUE_BLOCK - 1) / QUEUE_BLOCK;
    if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
    const dim3 grid((unsigned)blocks);
    const uint64_t rings = queue_rings_bytes(job);
    if (job->model == CIMBA_B200_MODEL_GG1) {
        if (job->variant == 1) return launch_kernel(job, queue_kernel<1, false>, queue_kernel<1, true>, grid, QUEUE_BLOCK, 0, st, qa, "queue_kernel launch");
        return then_repair<models::GG1>(launch_kernel(job, gg1_kernel<false>, gg1_kernel<true>, grid, QUEUE_BLOCK, 0, st, qa, "gg1_kernel launch"),
                                        job, rings, st, "repair pass (G/G/1)");
    }
    if (job->model == CIMBA_B200_MODEL_MM1_RECORDED) {
        if (job->counters == nullptr)
            return fail(CIMBA_B200_EINVAL, "CIMBA_B200_MODEL_MM1_RECORDED writes its cmb_wtdsummary to counters[]");
        const int e = launch_kernel(job, queue_kernel<0, false, true>, queue_kernel<0, true, true>, grid, QUEUE_BLOCK, 0, st, qa,
                                    "queue_kernel (recorded) launch");
        return then_repair<models::MM1Recorded>(e, job, rings, st, "repair pass (M/M/1 with its queue history)");
    }
    if (job->variant == 1) return launch_kernel(job, queue_kernel<0, false>, queue_kernel<0, true>, grid, QUEUE_BLOCK, 0, st, qa, "queue_kernel launch");
    int e;
    if (job->variant == 2) {                        // variates from producer warps (mm1_pc.cuh): an experiment, same answers
        if (mapping != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "variant 2 of MODEL_MM1 runs one trial per lane");
        const dim3 pc_grid((unsigned)((job->num_trials + MM1_PC_CONSUMERS - 1) / MM1_PC_CONSUMERS));
        e = launch_kernel(job, mm1_pc_kernel<false>, mm1_pc_kernel<true>, pc_grid, 2 * MM1_PC_CONSUMERS, 0, st, qa, "mm1_kernel launch");
    }
    else {
        if (const int c = mm1_prefer_shared()) return c;
        e = launch_kernel(job, mm1_kernel<false>, mm1_kernel<true>, grid, QUEUE_BLOCK, 0, st, qa, "mm1_kernel launch");
    }
    return then_repair<models::MM1>(e, job, rings, st, "repair pass (M/M/1)");
}

int mmc_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (job->servers < 1) return fail(CIMBA_B200_EINVAL, "servers must be >= 1 for CIMBA_B200_MODEL_MMC");
    if (mapping_of(job) != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "MODEL_MMC supports CIMBA_B200_MAP_LANE only");
    if (const int e = check_workspace(job)) return e;
    PoolArgs pa = cmb::job_args<PoolArgs>(*job);
    pa.servers = job->servers;
    pa.num_objects = job->num_objects;
    pa.arr_mean = job->arr_mean;
    pa.srv_mean = job->srv_mean;
    pa.spill = (double *)job->workspace;
    pa.spill_cap = cmb::spill_cap(*job);
    pa.diag = (unsigned long long *)job->diag;
    const uint64_t blocks = (job->num_trials + POOL_BLOCK - 1) / POOL_BLOCK;
    if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
    const bool readable = job->variant == 1;        // the readable formulation, pool_model.cuh
    const int e = launch_kernel(job, readable ? pool_kernel<false> : pool_fast_kernel<false>, readable ? pool_kernel<true> : pool_fast_kernel<true>,
                                dim3((unsigned)blocks), POOL_BLOCK, 0, st, pa, "pool_kernel launch");
    return then_repair<models::MMC>(e, job, queue_rings_bytes(job), st, "repair pass (M/M/c)");
}

// ---- the reference's own test worlds (models 3-6, 8, 11-14): a fixed-capacity kernel each (csrc/general.cuh, faster than
// the engine) behind which the general engine re-runs whatever that kernel flags
bool has_capacity(const cimba_b200_device_job *job)
{
    return job->model != CIMBA_B200_MODEL_TIMERS && job->model != CIMBA_B200_MODEL_RESOURCE_RECORDED;
}

template <bool TRACE>
auto coverage_kernel(int m)
{
    return m == CIMBA_B200_MODEL_RESOURCE_RECORDED ? resource_kernel<TRACE>
         : m == CIMBA_B200_MODEL_TIMERS ? timers_kernel<TRACE>
         : m == CIMBA_B200_MODEL_PRIOQ ? prioq_kernel<TRACE>
         : m == CIMBA_B200_MODEL_BUFFER || m == CIMBA_B200_MODEL_BUFFER_RECORDED ? buffer_kernel<TRACE>
         : m == CIMBA_B200_MODEL_PREEMPT ? preempt_kernel<TRACE>
                                         : guarded_kernel<TRACE>;
}

uint64_t coverage_workspace(const cimba_b200_device_job *job)
{
    return cmb::rings_then_arena(job->num_trials * (uint64_t)sizeof(GeneralState), repair_arena_bytes(job));
}

template <class Model>
int coverage_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    const int m = job->model;
    if (has_capacity(job) && job->servers < 1) return fail(CIMBA_B200_EINVAL, "capacity (servers) must be >= 1");
    if (mapping_of(job) != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "MODEL_GUARDED supports CIMBA_B200_MAP_LANE only");
    if (const int e = check_workspace(job)) return e;
    GuardedArgs ga = cmb::job_args<GuardedArgs>(*job);
    ga.capacity = job->servers;
    ga.duration = job->num_objects;
    ga.put_mean = job->arr_mean;
    ga.get_mean = job->srv_mean;
    ga.counters = job->counters;
    ga.state = (GeneralState *)job->workspace;
    ga.record = (m == CIMBA_B200_MODEL_GUARDED_RECORDED || m == CIMBA_B200_MODEL_BUFFER_RECORDED || m == CIMBA_B200_MODEL_PRIOQ_RECORDED) ? 1u : 0u;
    ga.use_pq = m == CIMBA_B200_MODEL_PRIOQ_RECORDED ? 1u : 0u;
    const uint64_t blocks = (job->num_trials + GUARDED_BLOCK - 1) / GUARDED_BLOCK;
    if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
    const int e = launch_kernel(job, coverage_kernel<false>(m), coverage_kernel<true>(m), dim3((unsigned)blocks), GUARDED_BLOCK, 0, st, ga,
                                "guarded_kernel launch");
    return then_repair<Model>(e, job, job->num_trials * (uint64_t)sizeof(GeneralState), st, "repair pass");
}

template <class Model>
int coverage_engine_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (const int e = engine_checks(job, has_capacity(job) ? "capacity (servers) must be >= 1" : nullptr)) return e;
    return launch_engine<Model>(job, st, "trial_kernel launch");
}

// CIMBA_B200_VARIANT_GENERAL, or more servers than the kernel's tables hold (max_servers), goes to the engine directly
template <class Model>
const Route *coverage_route(const cimba_b200_device_job *job, int max_servers)
{
    static constexpr Route fast{coverage_workspace, coverage_launch<Model>};
    static constexpr Route engine{engine_workspace<Model>, coverage_engine_launch<Model>};
    return job->variant == CIMBA_B200_VARIANT_GENERAL || job->servers > max_servers ? &engine : &fast;
}

// The static tier for the reference's queue tests (models 3, 6, 11 and 13): a job asks for the workspace of its default route -
// the fixed-capacity kernel's up to MAX servers, the general engine's above (coverage_route) - and the repair pass grows in all
// of it.  The object queue keeps its on-chip window and no HBM ring: one that outgrows the window flags the trial.
template <class Model, int MAX>
uint64_t coverage_or_engine_workspace(const cimba_b200_device_job *job)
{
    return job->servers > MAX ? engine_workspace<Model>(job) : coverage_workspace(job);
}

template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT>
int static_coverage_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (job->servers < 1) return fail(CIMBA_B200_EINVAL, "capacity (servers) must be >= 1");
    if (mapping_of(job) != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "the static tier runs one trial per lane (CIMBA_B200_MAP_LANE)");
    if (const int e = check_workspace(job)) return e;
    return counted(cmb::launch_static_trials<ModelT, NPROC, NQUEUE, NEVENT, false>(*job, st), "static_trial_kernel launch",
                   job->status != nullptr ? 2 : 1);
}

template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT, int MAX>
constexpr Route STATIC_COVERAGE{coverage_or_engine_workspace<ModelT<cmb::Sim>, MAX>, static_coverage_launch<ModelT, NPROC, NQUEUE, NEVENT>};

// ---- the harbor: up to 32 768 trials warp-per-trial with the state in shared memory, the rest lane-per-trial in HBM
uint64_t harbor_workspace(const cimba_b200_device_job *job) { return job->num_trials * (uint64_t)sizeof(HarborState); }

int harbor_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (job->servers < 3 || job->servers > 255)
        return fail(CIMBA_B200_EINVAL, "tugs (servers) must be in 3..255 for CIMBA_B200_MODEL_HARBOR (a large ship needs 3)");
    if (mapping_of(job) != CIMBA_B200_MAP_LANE) return fail(CIMBA_B200_EINVAL, "MODEL_HARBOR supports CIMBA_B200_MAP_LANE only");
    if (const int e = check_workspace(job)) return e;
    HarborArgs ha = cmb::job_args<HarborArgs>(*job);
    ha.tugs = job->servers;
    ha.duration = job->num_objects;
    ha.arr_mean = job->arr_mean;
    ha.unload_small = job->srv_mean;
    ha.counters = job->counters;
    ha.state = job->workspace;
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
        const void *fn = job->trace_cap > 0u ? (const void *)harbor_on_chip_kernel<true> : (const void *)harbor_on_chip_kernel<false>;
        CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        const uint64_t per_block = HARBOR_BLOCK_ON_CHIP / 32;
        unsigned nb = 0;
        if (const int e = resident_grid(fn, HARBOR_BLOCK_ON_CHIP, smem, 4, (job->num_trials + per_block - 1) / per_block, &nb)) return e;
        const int e = launch_kernel(job, harbor_on_chip_kernel<false>, harbor_on_chip_kernel<true>, dim3(nb), HARBOR_BLOCK_ON_CHIP, smem, st, ha,
                                    "harbor_on_chip_kernel launch");
        if (e != CIMBA_B200_OK || job->variant == 1) return e;
        ha.repair = 1u;
    }
    const uint64_t blocks = (job->num_trials + GUARDED_BLOCK - 1) / GUARDED_BLOCK;
    if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
    return launch_kernel(job, harbor_kernel<false>, harbor_kernel<true>, dim3((unsigned)blocks), GUARDED_BLOCK, 0, st, ha, "harbor_kernel launch");
}

// ---- AWACS: one trial per warp over the terrain registered for the device
uint64_t awacs_workspace(const cimba_b200_device_job *job) { return job->num_trials * (uint64_t)AWACS_STATE_BYTES; }

int awacs_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (job->num_objects == 0u) return fail(CIMBA_B200_EINVAL, "MODEL_AWACS: num_objects = trial duration in seconds, > 0");
    if (const int e = check_workspace(job)) return e;
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    AwacsArgs aa = cmb::job_args<AwacsArgs>(*job);
    {
        std::lock_guard<std::mutex> hold(g_terrain_mu);
        if (dev < 0 || dev >= MAX_TERRAIN_DEVICES || !g_terrain_set[dev])
            return fail(CIMBA_B200_EINVAL, "MODEL_AWACS: no terrain registered on this device; call cimba_b200_awacs_set_terrain()");
        aa.ter = g_terrain[dev];
    }
    aa.orbit = awacs_orbit();
    aa.t_end_s = (double)job->num_objects;
    aa.state = (unsigned char *)job->workspace;
    aa.counters = job->counters;
    const uint64_t per_block = AWACS_BLOCK / 32;
    const uint64_t blocks = (job->num_trials + per_block - 1) / per_block;
    if (blocks > 0x7fffffffull) return fail(CIMBA_B200_EINVAL, "too many trials for one launch");
    return launch_kernel(job, awacs_kernel<false>, awacs_kernel<true>, dim3((unsigned)blocks), AWACS_BLOCK, 0, st, aa, "awacs_kernel launch");
}

// ---- the hold model: variant 1 keeps the whole list in shared memory (hold_model.cuh); the others keep levels >= 2 of
// the 32-ary heap in HBM/L2 (hold_deep.cuh), with 32 (variant 2), 16 (3), 8 (4) or HOLD_DEFAULT_LANES (0) lanes per trial
uint64_t hold_workspace(const cimba_b200_device_job *job)
{
    return job->variant != 1 ? job->num_trials * deep_row_entries(job->servers) * (uint64_t)sizeof(uint4) : 0u;
}

template <bool TRACE>
auto deep_kernel(int lanes)
{
    return lanes == 32 ? hold_deep_kernel<TRACE> : lanes == 16 ? hold_group_kernel<16, TRACE> : hold_group_kernel<8, TRACE>;
}

int hold_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    const bool on_chip = job->variant == 1;
    if (job->servers < 1 || (on_chip && job->servers > HOLD_CAP - 8) ||
        (uint32_t)job->servers + 2u > DEEP_MAX_ENTRIES)
        return fail(CIMBA_B200_EINVAL, "workers (servers) must be in 1..33822 for CIMBA_B200_MODEL_HOLD (1..1080 with variant 1)");
    const bool trace = job->trace_cap > 0u;
    HoldArgs ha = cmb::job_args<HoldArgs>(*job);
    ha.workers = job->servers;
    ha.duration = job->num_objects;
    ha.mean = job->arr_mean;
    ha.counters = job->counters;
    unsigned blocks = 0;
    if (!on_chip) {
        if (const int e = check_workspace(job)) return e;
        const int lanes = job->variant == 2 ? 32 : (job->variant == 4 ? 8 : (job->variant == 3 ? 16 : HOLD_DEFAULT_LANES));
        const void *fn = trace ? (const void *)deep_kernel<true>(lanes) : (const void *)deep_kernel<false>(lanes);
        const uint64_t trials_per_block = (uint64_t)(DEEP_BLOCK / 32) * (uint64_t)(32 / lanes);
        if (const int e = resident_grid(fn, DEEP_BLOCK, 0, 8, (job->num_trials + trials_per_block - 1) / trials_per_block, &blocks)) return e;
        DeepArgs da{};
        da.h = ha;
        da.rows = (uint4 *)job->workspace;
        da.row_entries = deep_row_entries(job->servers);
        return launch_kernel(job, deep_kernel<false>(lanes), deep_kernel<true>(lanes), dim3(blocks), DEEP_BLOCK, 0, st, da, "hold_deep_kernel launch");
    }
    // persistent one-warp CTAs: exactly as many as are resident at once (shared memory
    // bounds it at ~12 per SM), so no CTA waits for another to retire
    const void *fn = trace ? (const void *)hold_kernel<true> : (const void *)hold_kernel<false>;
    if (const int e = resident_grid(fn, 32, HOLD_SMEM_BYTES, 8, job->num_trials, &blocks)) return e;
    return launch_kernel(job, hold_kernel<false>, hold_kernel<true>, dim3(blocks), 32, HOLD_SMEM_BYTES, st, ha, "hold_kernel launch");
}

// ---- a model loaded with cimba_b200_model_load
uint64_t user_workspace(const cimba_b200_device_job *job) { return user_model(job->model)->workspace_bytes(job); }

int user_launch(const cimba_b200_device_job *job, cudaStream_t st)
{
    if (const int e = check_workspace(job)) return e;
    const UserModel *um = user_model(job->model);
    return counted(um->launch(job, st), um->name.c_str());
}

constexpr Route QUEUE{queue_workspace, queue_launch};
constexpr Route MMC_FAST{queue_workspace, mmc_launch};
constexpr Route HARBOR{harbor_workspace, harbor_launch};
constexpr Route HARBOR_ENGINE{engine_workspace<models::HarborGeneral>, harbor_engine_launch};
constexpr Route AWACS{awacs_workspace, awacs_launch};
constexpr Route HOLD{hold_workspace, hold_launch};
constexpr Route USER{user_workspace, user_launch};

// The route that serves the job, nullptr for an unknown model
const Route *route(const cimba_b200_device_job *job)
{
    const bool general = job->variant == CIMBA_B200_VARIANT_GENERAL, on_static = job->variant == CIMBA_B200_VARIANT_STATIC;
    switch (job->model) {
    case CIMBA_B200_MODEL_MM1:          return on_static ? &STATIC<models::MM1T, 2, 1> : general ? &ENGINE<models::MM1> : &QUEUE;
    case CIMBA_B200_MODEL_GG1:          return on_static ? &STATIC<models::GG1T, 2, 1> : general ? &ENGINE<models::GG1> : &QUEUE;
    case CIMBA_B200_MODEL_MM1_RECORDED: return on_static ? &STATIC<models::MM1RecordedT, 2, 1> : general ? &ENGINE<models::MM1Recorded> : &QUEUE;
    case CIMBA_B200_MODEL_TUTORIAL1:    return general ? &ENGINE<models::Tutorial1> : &STATIC<models::Tutorial1T, 2, 0, 3>;
    case CIMBA_B200_MODEL_MMC:          return general || job->servers > 14 ? &ENGINE<models::MMC> : &MMC_FAST;
    case CIMBA_B200_MODEL_HOLD:         return general ? &ENGINE<models::HoldGeneral> : &HOLD;
    case CIMBA_B200_MODEL_HARBOR:       return general ? &HARBOR_ENGINE : &HARBOR;
    case CIMBA_B200_MODEL_AWACS:        return &AWACS;
    case CIMBA_B200_MODEL_RENEGE:       return &ENGINE<models::Renege>;
    case CIMBA_B200_MODEL_POOL_RECORDED:
        return on_static ? &STATIC_IN<models::CheeseT, 6, 6, engine_workspace<models::Cheese>, true> : &ENGINE<models::Cheese>;
    case CIMBA_B200_MODEL_PARK:         return &ENGINE<models::Park>;
    case CIMBA_B200_MODEL_TUTORIAL2:
        return on_static ? &STATIC_IN<models::Tutorial2T, 8, 8, engine_workspace<models::Tutorial2>, true> : &ENGINE<models::Tutorial2>;
    case CIMBA_B200_MODEL_GUARDED:
        return on_static ? &STATIC_COVERAGE<models::GuardedQueueT, 7, 1, 2, 16> : coverage_route<models::Guarded<false, false>>(job, 16);
    case CIMBA_B200_MODEL_GUARDED_RECORDED:
        return on_static ? &STATIC_COVERAGE<models::GuardedRecordedQueueT, 7, 1, 2, 16> : coverage_route<models::Guarded<false, true>>(job, 16);
    case CIMBA_B200_MODEL_PRIOQ_RECORDED:
        return on_static ? &STATIC_COVERAGE<models::GuardedPriorityQueueT, 7, 0, 2, 15> : coverage_route<models::Guarded<true, true>>(job, 15);
    case CIMBA_B200_MODEL_PRIOQ:
        return on_static ? &STATIC_COVERAGE<models::QueueAndTideT, 8, 0, 2, 15> : coverage_route<models::QueueAndTide>(job, 15);
    case CIMBA_B200_MODEL_PREEMPT:            // no table sized by `servers`
        return on_static ? &STATIC_IN<models::PoolFightT, 6, models::POOLFIGHT_SPARE_SLOTS, coverage_workspace, true>
                         : coverage_route<models::PoolFight>(job, INT32_MAX);
    case CIMBA_B200_MODEL_BUFFER:
        return on_static ? &STATIC_IN<models::WorkshopBufferT, 7, models::WORKSHOP_SPARE_SLOTS, coverage_workspace, true>
                         : coverage_route<models::Workshop<false>>(job, INT32_MAX);
    case CIMBA_B200_MODEL_BUFFER_RECORDED:
        return on_static ? &STATIC_IN<models::WorkshopRecordedT, 7, models::WORKSHOP_SPARE_SLOTS, coverage_workspace, true>
                         : coverage_route<models::Workshop<true>>(job, INT32_MAX);
    case CIMBA_B200_MODEL_TIMERS:
        return on_static ? &STATIC_IN<models::FrontDeskT, 8, models::FRONTDESK_SPARE_SLOTS, coverage_workspace, false>
                         : coverage_route<models::FrontDesk>(job, INT32_MAX);
    case CIMBA_B200_MODEL_RESOURCE_RECORDED:
        return on_static ? &STATIC_IN<models::ToolT, 4, 2, coverage_workspace, false> : coverage_route<models::Tool>(job, INT32_MAX);
    }
    return job->model >= CIMBA_B200_MODEL_USER_BASE && user_model(job->model) != nullptr ? &USER : nullptr;
}

}  // namespace

extern "C" {

const char *cimba_b200_version(void) { return CIMBA_B200_VERSION_STRING; }
const char *cimba_b200_last_error(void) { return g_err; }
uint64_t cimba_b200_launch_count(void) { return g_launches.load(); }

int cimba_b200_mm1_resident_ctas(int trace)
{
    if (const int e = mm1_prefer_shared()) return e;
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, trace ? mm1_kernel<true> : mm1_kernel<false>, QUEUE_BLOCK, 0));
    return per_sm;
}

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
    const Route *r = job != nullptr ? route(job) : nullptr;
    return r != nullptr ? r->workspace(job) : 0u;
}

int cimba_b200_launch(const cimba_b200_device_job *job, void *stream)
{
    if (job == nullptr) return fail(CIMBA_B200_EINVAL, "job is NULL");
    if (job->num_trials == 0u) return fail(CIMBA_B200_EINVAL, "num_trials must be > 0 (src/cimba.c:157)");
    if ((job->arr_mean == nullptr || job->srv_mean == nullptr) && job->model != CIMBA_B200_MODEL_AWACS)
        return fail(CIMBA_B200_EINVAL, "arr_mean/srv_mean device arrays are required");
    if (job->num_objects >= 0xffffffffull) return fail(CIMBA_B200_EINVAL, "num_objects must be < 2^32-1");
    const int mapping = mapping_of(job);
    if (mapping != CIMBA_B200_MAP_LANE && mapping != CIMBA_B200_MAP_WARP)
        return fail(CIMBA_B200_EINVAL, "mapping must be CIMBA_B200_MAP_LANE or CIMBA_B200_MAP_WARP");
    if (job->trace_cap > 0u && (job->trace_key == nullptr || job->trace_time == nullptr))
        return fail(CIMBA_B200_EINVAL, "trace_cap > 0 needs trace_key and trace_time");
    if (cimba_b200_device_count() <= 0) return fail(CIMBA_B200_ENODEVICE, "no CUDA device");
    if (cmb::spill_cap(*job) == 0u)
        return fail(CIMBA_B200_EINVAL, "queue_spill_cap must be 0 (default) or a power of two <= 2^26");
    if (job->num_params > CIMBA_B200_MAX_MODEL_PARAMS || (job->num_params > 0u && job->params == nullptr))
        return fail(CIMBA_B200_EINVAL, "params: at most CIMBA_B200_MAX_MODEL_PARAMS doubles behind a HOST pointer");

    const Route *r = route(job);
    if (r == nullptr)
        return fail(CIMBA_B200_EINVAL, job->model >= CIMBA_B200_MODEL_USER_BASE
                                           ? "unknown model id (cimba_b200_model_load returns the ids of loaded models)" : "unknown model");
    return r->launch(job, (cudaStream_t)stream);
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
// The trials [lo, hi) of `job` as a job of their own: its arrays offset into the job's, seeds from the global trial index
cimba_b200_device_job sub_job(const cimba_b200_device_job &job, uint64_t lo, uint64_t hi)
{
    cimba_b200_device_job s = job;
    s.first_trial = job.first_trial + lo;
    s.num_trials = hi - lo;
    s.arr_mean = job.arr_mean + lo;
    s.srv_mean = job.srv_mean + lo;
    s.events = job.events + lo;
    s.objects = job.objects + lo;
    s.t_end = job.t_end + lo;
    s.sum_wait = job.sum_wait + lo;
    s.status = job.status + lo;
    s.max_queue = job.max_queue + lo;
    s.counters = job.counters + 8u * lo;
    return s;
}

// Re-run the trials of `job` whose status (host copy in `status`, kept up to date) says the growth arena ran out.  The
// arena is shared by every trial of a launch and never reclaimed, so its need grows with the trial count: the run from the
// first such trial to the last goes again (in one launch; the clean trials in it give what they gave) with 4x the workspace
// its size asks for, then 4x more per round, up to half of the device's free memory; past that the run is split in halves.  Seeds follow the global trial index, so what comes back
// is what one launch with room enough would have given.  A trial that still cannot fit keeps its flag.
int rerun_exhausted(const cimba_b200_device_job &job, uint32_t *status, cudaStream_t st)
{
    struct Run { uint64_t lo, hi, ws; };
    std::vector<Run> todo;
    auto collect = [&](uint64_t lo, uint64_t hi, uint64_t ws) {     // one run from the first such trial to the last
        while (lo < hi && (status[lo] & CIMBA_B200_TRIAL_ARENA_EXHAUSTED) == 0u) lo++;
        while (hi > lo && (status[hi - 1u] & CIMBA_B200_TRIAL_ARENA_EXHAUSTED) == 0u) hi--;
        if (lo < hi) todo.push_back({lo, hi, ws});
    };
    collect(0u, job.num_trials, 0u);
    while (!todo.empty()) {
        const Run r = todo.back();
        todo.pop_back();
        cimba_b200_device_job s = sub_job(job, r.lo, r.hi);
        size_t free_bytes = 0, total_bytes = 0;
        CUDA_TRY(cudaMemGetInfo(&free_bytes, &total_bytes));
        const uint64_t cap = free_bytes / 2u;
        const uint64_t least = cimba_b200_workspace_bytes(&s);
        uint64_t ws = r.ws != 0u ? r.ws : 4u * least;
        if (ws > cap) ws = cap;
        if (ws <= least) continue;                      // no room for more than the first launch had: the flag stays
        void *mem = nullptr;
        CUDA_TRY(cudaMalloc(&mem, ws));
        s.workspace = mem;
        s.workspace_bytes = ws;
        int rc = cimba_b200_launch(&s, st);
        cudaError_t e = cudaSuccess;
        if (rc == CIMBA_B200_OK) {
            e = cudaMemcpyAsync(status + r.lo, s.status, (r.hi - r.lo) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        }
        cudaFree(mem);
        if (rc != CIMBA_B200_OK) return rc;
        if (e != cudaSuccess) return cuda_fail(e, "re-run of exhausted trials");
        if (ws < cap) {
            collect(r.lo, r.hi, ws < cap / 4u ? 4u * ws : cap);
        }
        else if (r.hi - r.lo > 1u) {                    // at the cap: fewer trials share the arena
            const uint64_t mid = r.lo + (r.hi - r.lo) / 2u;
            collect(r.lo, mid, cap);
            collect(mid, r.hi, cap);
        }
    }
    return CIMBA_B200_OK;
}

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
        uint32_t *stt = (uint32_t *)(sw + n);
        const uint32_t *mq = stt + n;
        bool exhausted = false;
        for (uint64_t i = 0; i < n && !exhausted; i++) exhausted = (stt[i] & CIMBA_B200_TRIAL_ARENA_EXHAUSTED) != 0u;
        if (exhausted) {                                // more workspace for the trials that ran out, then the results again
            rc = rerun_exhausted(job, stt, st);
            if (rc != CIMBA_B200_OK) goto done;
            e = cudaMemcpyAsync(h_out, d_out, out_bytes + (want_counters ? cnt_bytes : 0), cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            if (e != cudaSuccess) { rc = cuda_fail(e, "D2H after re-run"); goto done; }
            clk.lap("re-run of exhausted trials");
        }
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

double cimba_b200_datasummary_variance(const cimba_b200_datasummary *s) { return summary_variance(*s); }
double cimba_b200_datasummary_stddev(const cimba_b200_datasummary *s) { return summary_stddev(*s); }

uint64_t cimba_b200_datasummary_count(const cimba_b200_datasummary *s) { return s->count; }
double cimba_b200_datasummary_max(const cimba_b200_datasummary *s) { return s->max; }
double cimba_b200_datasummary_min(const cimba_b200_datasummary *s) { return s->min; }

double cimba_b200_datasummary_skewness(const cimba_b200_datasummary *s) { return summary_skewness(*s); }
double cimba_b200_datasummary_kurtosis(const cimba_b200_datasummary *s) { return summary_kurtosis(*s); }

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
