// cmb_launch.cuh - host side of a model built on cmb_device.cuh: fill the kernel's arguments from the C-ABI job,
// size and reset the growth arena, launch.  Used by the library itself (its built-in general-engine models and the
// repair pass of the fast kernels) and, through CMB_EXPORT_MODEL, by a model compiled into a library of its own.
#pragma once

#include <cstdio>
#include <cstring>
#include <cuda_runtime.h>

#include "../../include/cimba_b200.h"
#include "cmb_kernel.cuh"
#include "cmb_static.cuh"

namespace cimba_b200 {
namespace cmb {

// Growth memory of a launch.  A model may say what a trial needs (static uint64_t arena_bytes_per_trial(const
// cimba_b200_device_job &)); the default suits models with a handful of processes.
template <class Model, class = void>
struct ArenaNeed {
    static uint64_t per_trial(const cimba_b200_device_job &) { return 32768u; }
};
template <class Model>
struct ArenaNeed<Model, decltype((void)Model::arena_bytes_per_trial(*(const cimba_b200_device_job *)nullptr))> {
    static uint64_t per_trial(const cimba_b200_device_job &job) { return Model::arena_bytes_per_trial(job); }
};

#ifndef CMB_RESIDENT_CTAS
// CTAs of CMB_BLOCK threads per SM at most.  Each trial's control block is a ~2 KB stack frame, so this bounds the local-memory
// working set: on an H100 (50 MB L2, 132 SMs), M/M/1 on the general engine at 65 536 trials ran at 1.66e9 events/s with 4,
// 1.18e9 with 8 or 16 (all trials resident at once), same answers.
#define CMB_RESIDENT_CTAS 4u
#endif

constexpr uint64_t ARENA_HEADER = 256u;         // the allocation cursor lives in front of the arena

// What a fixed-capacity kernel flags (its queue, event list, wait lists or process table outgrew their tables) is re-run
// on the general engine, whose containers grow, by a repair pass inside the same launch.
constexpr uint32_t REPAIR_BITS = CIMBA_B200_TRIAL_QUEUE_OVERFLOW | CIMBA_B200_TRIAL_FEL_OVERFLOW |
                                 CIMBA_B200_TRIAL_GUARD_OVERFLOW | CIMBA_B200_TRIAL_PROC_OVERFLOW;

constexpr uint32_t SPILL_CAP_DEFAULT = 512u;    // HBM ring entries per queue and trial behind the on-chip window

// job.queue_spill_cap: 0 = the default, else a power of two up to 2^26; 0 = invalid
inline uint32_t spill_cap(const cimba_b200_device_job &job)
{
    const uint64_t c = job.queue_spill_cap;
    if (c == 0u) return SPILL_CAP_DEFAULT;
    return (c & (c - 1u)) == 0u && c <= (1ull << 26) ? (uint32_t)c : 0u;
}

inline uint64_t align256(uint64_t v) { return (v + 255u) & ~(uint64_t)255u; }

// The workspace of a fixed-capacity kernel: its rings, then (256-byte aligned) the growth arena of its repair pass
inline uint64_t rings_then_arena(uint64_t rings_bytes, uint64_t arena_bytes) { return align256(rings_bytes) + arena_bytes; }

// The fields every kernel argument struct has, from the job; the caller fills the rest
template <class Args>
Args job_args(const cimba_b200_device_job &job)
{
    Args a{};
    a.master_seed = job.master_seed;
    a.first_trial = job.first_trial;
    a.num_trials = job.num_trials;
    a.events = job.events;
    a.objects = job.objects;
    a.t_end = job.t_end;
    a.sum_wait = job.sum_wait;
    a.status = job.status;
    a.max_queue = job.max_queue;
    a.trace_cap = job.trace_cap;
    a.trace_key = job.trace_key;
    a.trace_time = job.trace_time;
    return a;
}

inline LaunchArgs launch_args(const cimba_b200_device_job &job)
{
    LaunchArgs a = job_args<LaunchArgs>(job);
    a.num_objects = job.num_objects;
    a.servers = job.servers;
    a.arr_mean = job.arr_mean;
    a.srv_mean = job.srv_mean;
    a.counters = job.counters;
    a.diag = (unsigned long long *)job.diag;
    a.num_params = job.params != nullptr ? (job.num_params < 16u ? job.num_params : 16u) : 0u;
    for (uint32_t k = 0; k < a.num_params; k++) a.params[k] = job.params[k];
    return a;
}

template <class Model>
uint64_t workspace_bytes_for(const cimba_b200_device_job &job)
{
    return ARENA_HEADER + job.num_trials * ArenaNeed<Model>::per_trial(job) + (64ull << 20);
}

// Launch Model over the job's trials on `stream`, growth arena = [arena, arena + arena_bytes) (device memory, 256-byte
// aligned; the first ARENA_HEADER bytes hold the cursor).  only_flagged = 0: every trial; else the repair pass.
// Returns a cudaError_t as int (0 = launched).
template <class Model>
int launch_model(const cimba_b200_device_job &job, unsigned char *arena, uint64_t arena_bytes, uint32_t only_flagged,
                 cudaStream_t stream)
{
    if (arena == nullptr || arena_bytes <= ARENA_HEADER) return (int)cudaErrorInvalidValue;
    LaunchArgs a = launch_args(job);
    a.only_flagged = only_flagged;
    a.arena_base = arena;
    a.arena_bytes = arena_bytes - ARENA_HEADER;

    cudaError_t e = cudaMemsetAsync(arena, 0, ARENA_HEADER, stream);
    if (e != cudaSuccess) return (int)e;
    const bool trace = job.trace_cap > 0u;
    const void *fn = trace ? (const void *)trial_kernel<Model, true> : (const void *)trial_kernel<Model, false>;
    // the per-trial control block (cmb::Sim + the model) is the kernel's stack frame: make room for it
    cudaFuncAttributes attr{};
    e = cudaFuncGetAttributes(&attr, fn);
    if (e != cudaSuccess) return (int)e;
    size_t limit = 0;
    (void)cudaDeviceGetLimit(&limit, cudaLimitStackSize);
    if (attr.localSizeBytes + 1024u > limit) {
        e = cudaDeviceSetLimit(cudaLimitStackSize, attr.localSizeBytes + 1024u);
        if (e != cudaSuccess) return (int)e;
    }
    int dev = 0, sms = 132;
    (void)cudaGetDevice(&dev);
    (void)cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const uint64_t wanted = (job.num_trials + CMB_BLOCK - 1) / CMB_BLOCK;
    const uint64_t resident = (uint64_t)sms * CMB_RESIDENT_CTAS;   // trials beyond that are taken grid-stride
    const unsigned blocks = (unsigned)(wanted < resident ? wanted : resident);
    void *kargs[] = { (void *)&a };
    e = cudaLaunchKernel(fn, dim3(blocks), dim3(CMB_BLOCK), kargs, 0, stream);
    if (e != cudaSuccess) return (int)e;
    return (int)cudaGetLastError();
}

// The repair pass behind a fixed-capacity kernel whose rings take `rings_bytes` at the front of the workspace
template <class Model>
int launch_repair(const cimba_b200_device_job &job, uint64_t rings_bytes, uint64_t arena_bytes, cudaStream_t stream)
{
    return launch_model<Model>(job, (unsigned char *)job.workspace + align256(rings_bytes), arena_bytes, REPAIR_BITS, stream);
}

// ---- the static tier (cmb_static.cuh): ModelT<StaticSim<NPROC, NQUEUE>> first, ModelT<Sim> for what it flags
inline uint64_t static_rings_bytes(const cimba_b200_device_job &job, int nqueue)
{
    return align256(job.num_trials * (uint64_t)nqueue * spill_cap(job) * sizeof(double));
}

template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT = 0>
uint64_t workspace_bytes_static(const cimba_b200_device_job &job)
{
    // the growth arena of the repair pass holds a share of the trials, not all of them
    const uint64_t arena = ARENA_HEADER + (job.num_trials / 8u + 256u) * ArenaNeed<ModelT<Sim>>::per_trial(job) + (64ull << 20);
    return rings_then_arena(static_rings_bytes(job, NQUEUE), arena);
}

// The static kernel over the job's trials, then the repair pass in the workspace behind its rings: launch_static_model below,
// or a route of the library that sizes the workspace itself (capi.cu).  RINGS = false: the queues keep only their on-chip
// window (a bounded queue that outgrows it flags the trial) and the whole workspace is the repair pass's.
template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT = 0, bool RINGS = true>
int launch_static_trials(const cimba_b200_device_job &job, cudaStream_t stream)
{
    const uint32_t cap = spill_cap(job);
    const uint64_t rings = RINGS ? static_rings_bytes(job, NQUEUE) : 0u;
    if (cap == 0u || job.workspace == nullptr || job.workspace_bytes <= rings + ARENA_HEADER) return (int)cudaErrorInvalidValue;
    StaticArgs sa{};
    sa.base = launch_args(job);
    sa.spill = RINGS ? (double *)job.workspace : nullptr;
    sa.spill_cap = RINGS ? cap : 0u;
    const uint64_t blocks = (job.num_trials + STATIC_BLOCK - 1) / STATIC_BLOCK;
    if (blocks == 0u || blocks > 0x7fffffffull) return (int)cudaErrorInvalidValue;
    const bool trace = job.trace_cap > 0u;
    const void *fn = trace ? (const void *)static_trial_kernel<ModelT, NPROC, NQUEUE, NEVENT, true>
                           : (const void *)static_trial_kernel<ModelT, NPROC, NQUEUE, NEVENT, false>;
    void *kargs[] = { (void *)&sa };
    cudaError_t e = cudaLaunchKernel(fn, dim3((unsigned)blocks), dim3(STATIC_BLOCK), kargs, 0, stream);
    if (e != cudaSuccess) return (int)e;
    e = cudaGetLastError();
    if (e != cudaSuccess || job.status == nullptr) return (int)e;      // nobody could see a flag: nothing to repair by
    return launch_repair<ModelT<Sim>>(job, rings, job.workspace_bytes - rings, stream);
}

template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT = 0>
int launch_static_model(const cimba_b200_device_job &job, cudaStream_t stream)
{
    if (spill_cap(job) == 0u || job.workspace == nullptr || job.workspace_bytes < workspace_bytes_static<ModelT, NPROC, NQUEUE, NEVENT>(job))
        return (int)cudaErrorInvalidValue;
    return launch_static_trials<ModelT, NPROC, NQUEUE, NEVENT>(job, stream);
}

}  // namespace cmb
}  // namespace cimba_b200

// A model template of the static tier in a library of its own: ModelT<cmb::StaticSim<NPROC, NQUEUE>> runs first, and
// ModelT<cmb::Sim> re-runs what that flags
#define CMB_EXPORT_STATIC_MODEL(ModelT, NPROC, NQUEUE, name_string) CMB_EXPORT_STATIC_MODEL_EVENTS(ModelT, NPROC, NQUEUE, 0, name_string)
// ... with NEVENT slots for events of the model's own (cmb_event_schedule), which also makes the event list order by priority
#define CMB_EXPORT_STATIC_MODEL_EVENTS(ModelT, NPROC, NQUEUE, NEVENT, name_string)                                    \
    extern "C" const char *cimba_b200_user_model_name(void) { return name_string; }                                  \
    extern "C" uint64_t cimba_b200_user_model_workspace_bytes(const cimba_b200_device_job *job)                      \
    {                                                                                                                 \
        return job ? cimba_b200::cmb::workspace_bytes_static<ModelT, NPROC, NQUEUE, NEVENT>(*job) : 0u;               \
    }                                                                                                                 \
    extern "C" int cimba_b200_user_model_launch(const cimba_b200_device_job *job, void *stream)                      \
    {                                                                                                                 \
        if (job == nullptr || job->workspace == nullptr) return (int)cudaErrorInvalidValue;                          \
        return cimba_b200::cmb::launch_static_model<ModelT, NPROC, NQUEUE, NEVENT>(*job, (cudaStream_t)stream);       \
    }

// A model in a library of its own: the three C entry points cimba_b200_model_load() looks up.
#define CMB_EXPORT_MODEL(Model, name_string)                                                                          \
    extern "C" const char *cimba_b200_user_model_name(void) { return name_string; }                                  \
    extern "C" uint64_t cimba_b200_user_model_workspace_bytes(const cimba_b200_device_job *job)                      \
    {                                                                                                                 \
        return job ? cimba_b200::cmb::workspace_bytes_for<Model>(*job) : 0u;                                          \
    }                                                                                                                 \
    extern "C" int cimba_b200_user_model_launch(const cimba_b200_device_job *job, void *stream)                      \
    {                                                                                                                 \
        if (job == nullptr || job->workspace == nullptr) return (int)cudaErrorInvalidValue;                          \
        return cimba_b200::cmb::launch_model<Model>(*job, (unsigned char *)job->workspace, job->workspace_bytes, 0u,  \
                                                    (cudaStream_t)stream);                                            \
    }
