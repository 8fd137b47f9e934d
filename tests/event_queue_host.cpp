// tests/event_queue_host.cpp - TEST INFRASTRUCTURE: the event list's queries, clear and pattern calls, compiled for the CPU from the
// SAME source text on both engines - examples/event_model.cuh's EventTestT and EventChurnT, plus this file's EdgeT - on the general
// engine (cimba_b200/csrc/cmb_device.cuh) and on cmb::StaticSimOf<ModelT, NPROC, NQUEUE, NEVENT> (cimba_b200/csrc/cmb_static.cuh),
// exported as a small C library for tests/test_event_queue.py.  EventTestT on the general engine also prints the text the reference's
// test/test_event.c prints, its event-list dumps read from the engine's heap array.  The CUDA vocabulary is mapped to C++ as in
// tests/cmb_engine_host.cpp.  Not a product path: built by the test.
//
// Build: g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC event_queue_host.cpp -o libevent_queue_host.so
#include <cinttypes>
#include <cstdarg>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
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

#include "../examples/event_model.cuh"

using namespace cimba_b200;
using namespace event_example;

// ---------------------------------------------------------------- the reference's text (test/test_event.c), from EventTestT's notes
static std::string g_text;
static uint32_t g_flag_point;           // the static run: the first dump point at which the trial was flagged (99 = never)

static void say(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
static void say(const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_text += buf;
}

static void line_of(char c)                     // cmi_test_print_line, test/test.h
{
    g_text.append(80, c);
    g_text += '\n';
}

static const char *name_of(uint32_t v)          // evstrs, and NULL as the reference's formatter shows it
{
    static const char *const ev[] = {"foo", "bar", "yuk"};
    return v == cmb::NIL ? "<NULL>" : v < 3u ? ev[v] : "?";
}

static void dump(const cmb::Sim &sim)           // cmb_event_queue_print with test_event.c's formatter: the heap array from slot 1
{
    say("--------------------- Event queue ---------------------\n");
    for (uint32_t k = 1u; k <= sim.fel.count; k++) {
        const cmb::Tag &t = sim.fel.tag[k];
        say("time %#8.4g prio %" PRIi64 ": hash_key %" PRIu64 "\t%s\t%s\t%s\n", t.d, (int64_t)t.prio, t.key,
            t.act == EventTestT<cmb::Sim>::TEST_ACTION ? "test_action" : "end_sim", name_of(t.subj), name_of((uint32_t)t.arg));
    }
    say("-------------------------------------------------------\n");
}

static void action_line(double now, const char *fn, int line, const char *msg)     // cmb_logger_user from the dispatcher
{
    say("%#10.5g\tdispatcher\t%s (%d):  %s\n", now, fn, line, msg);
}

struct PrintNote {
    static void at(cmb::Sim &sim, uint32_t what, uint64_t a, double t, int64_t p)
    {
        static const char *const after[7] = {
            "",
            "\nWildcard search, searching for test action events with subject yuk, any object\n",
            "\nScheduling new events with subject yuk\n",
            "\nRescheduling and reprioritizing two events with subject yuk\n",
            "\nWildcard search, counting events with subject bar, any object\n",
            "\nWildcard search, cancelling any events with subject bar, any object\n",
            "",
        };
        switch (what) {
        case NOTE_START:
            line_of('-');
            say("Testing event queue\nCreating queue, start time %g\nCurrent simulation time %g\nScheduling 3x3 events\n", t, sim.now);
            break;
        case NOTE_SCHEDULED: say("Scheduled event %" PRIu64 "\n", a); break;
        case NOTE_QUEUE:
            if (a == 0u) say("Scheduling end event\n");
            if (a == 1u) say("\nSearching for it again...  ");
            dump(sim);
            say("%s", after[a]);
            break;
        case NOTE_FOUND:
            say("\nSearching for an event (test_action\tbar\tfoo)...found event %" PRIu64 "\n", a);
            say("It has time %g priority %" PRIi64 ".\nCanceling it\n", t, p);
            break;
        case NOTE_CANCELING: say("\tcanceling %" PRIu64 "\n", a); break;
        case NOTE_COUNTED: say("Found %" PRIu64 " events\n", a); break;
        case NOTE_CANCELLED: say("Cancelled %" PRIu64 " events\n", a); break;
        case NOTE_EXECUTE:
            say("\nExecuting the simulation, starting time %#g\n", t);
            line_of('-');
            say("Time:\t\tType:\tAction: \t\tSubject:\t\tObject:\n");
            break;
        case NOTE_ACTION: {
            char msg[128];
            const bool test = a == EventTestT<cmb::Sim>::TEST_ACTION;
            snprintf(msg, sizeof msg, "%s\t%s\t%s", test ? "test_action" : "end_sim", name_of((uint32_t)p), name_of((uint32_t)(int64_t)t));
            action_line(sim.now, test ? "test_action" : "end_sim", test ? 45 : 55, msg);
            if (!test) action_line(sim.now, "end_sim", 56, "===> end_sim: game over <===");
            break;
        }
        }
    }
};

// the static run prints nothing (the tier has no heap array); it notes where the trial was first flagged
struct FlagNote {
    template <class S>
    static void at(S &sim, uint32_t what, uint64_t a, double, int64_t)
    {
        if (what == NOTE_QUEUE && g_flag_point == 99u && (sim.status & TRIAL_ERR_PROC_OVERFLOW) != 0u) g_flag_point = (uint32_t)a;
    }
};

template <class S> using EventTestPrinted = EventTestT<S, PrintNote>;
template <class S> using EventTestFlagged = EventTestT<S, FlagNote>;

// ---------------------------------------------------------------- EdgeT: one corner of the new calls per case (params[0])
//   0  cmb_event_time / _priority of a cancelled handle (BAD_ARGUMENT, 0), then of a live one
//   1  patterns next to process wake-ups: wildcard subjects never match one, a process index as subject does not either
//   2  CMB_ANY_SUBJECT and NIL are different subjects
//   3  cmb_event_queue_clear while a process waits on an event: nobody woken, the handle "not scheduled", keys run on
//   4  cmb_event_queue_initialize before the first schedule (the clock moves) and after it (flagged, the clock stays)
template <class S>
struct EdgeT {
    enum : uint32_t { USER = cmb::ACT_CMB_USER, CLEAR, AFTER };
    static constexpr bool static_interrupts = true;
    static constexpr bool static_waits = true;
    uint64_t counter[8];
    uint64_t awaited;
    uint32_t which;

    CMB_FN bool demand(S &, uint32_t, uint32_t, int32_t) { return false; }

    CMB_FN void process(S &sim, uint32_t me, uint32_t, int64_t sig)
    {
        EdgeT &m = *this;
        CMB_PROCESS_BEGIN
        if (which == 3u) {
            CMB_PROCESS_WAIT_EVENT(awaited);
            counter[7] = 100u + (uint64_t)sig;          // never: the event it waits on is dropped by the clear
        }
        else {
            CMB_PROCESS_HOLD(1.0);
        }
        CMB_PROCESS_END
    }

    CMB_FN void event(S &sim, uint32_t act, uint32_t, int64_t)
    {
        if (act == CLEAR) {
            cmb_event_queue_clear();
            counter[1] = cmb_event_current();
            counter[2] = cmb_event_queue_count() + (cmb_event_queue_is_empty() ? 10u : 0u);
            counter[4] = cmb_event_schedule(AFTER, 0, 0, __dadd_rn(cmb_time(), 1.0), 0);    // the reference cancels in a non-empty list only
            counter[3] = (cmb_event_is_scheduled(awaited) ? 1u : 0u) + (cmb_event_cancel(awaited) ? 10u : 0u);
        }
        else if (act == AFTER) {
            counter[5] = cmb_process_status(0u) + 10u * cmb_event_queue_count();
        }
    }

    CMB_FN void run_trial(S &sim, const cmb::TrialIn &in)
    {
        for (int k = 0; k < 8; k++) counter[k] = 0u;
        which = (uint32_t)in.params[0];
        awaited = 0u;
        if (which == 0u) {
            const uint64_t h = cmb_event_schedule(USER, 0, 0, 5.0, 1);
            (void)cmb_event_cancel(h);
            counter[0] = (uint64_t)__double_as_longlong(cmb_event_time(h));
            counter[1] = (uint64_t)cmb_event_priority(h);
            counter[2] = sim.status;
            const uint64_t live = cmb_event_schedule(USER, 0, 0, 7.0, -4);
            counter[3] = (uint64_t)__double_as_longlong(cmb_event_time(live));
            counter[4] = (uint64_t)cmb_event_priority(live);
        }
        else if (which == 1u) {
            cmb_process_start(cmb_process_create(0u, 0, 0u));
            cmb_process_start(cmb_process_create(0u, 0, 1u));
            counter[0] = cmb_event_pattern_count(CMB_ANY_ACTION, CMB_ANY_SUBJECT, CMB_ANY_OBJECT);
            counter[1] = cmb_event_pattern_find(CMB_ANY_ACTION, 0u, CMB_ANY_OBJECT);
            counter[2] = cmb_event_pattern_cancel(CMB_ANY_ACTION, 1u, CMB_ANY_OBJECT);
            counter[3] = cmb_event_queue_count();
            const uint64_t h = cmb_event_schedule(USER, 0u, 0, 0.5, 0);
            counter[4] = cmb_event_pattern_count(CMB_ANY_ACTION, 0u, CMB_ANY_OBJECT);
            counter[5] = cmb_event_pattern_find(CMB_ANY_ACTION, 0u, 0) == h ? 1u : 0u;
            counter[6] = cmb_event_pattern_cancel(CMB_ANY_ACTION, CMB_ANY_SUBJECT, CMB_ANY_OBJECT) + 10u * cmb_event_queue_count();
        }
        else if (which == 2u) {
            const uint64_t hn = cmb_event_schedule(USER, cmb::NIL, cmb::NIL, 1.0, 0);
            (void)cmb_event_schedule(USER, 5u, 7, 2.0, 0);
            counter[0] = cmb_event_pattern_count(CMB_ANY_ACTION, cmb::NIL, CMB_ANY_OBJECT);
            counter[1] = cmb_event_pattern_count(CMB_ANY_ACTION, CMB_ANY_SUBJECT, CMB_ANY_OBJECT);
            counter[2] = cmb_event_pattern_count(USER, cmb::NIL, cmb::NIL);
            counter[3] = cmb_event_pattern_count(USER, CMB_ANY_SUBJECT, 7);
            counter[4] = cmb_event_pattern_find(CMB_ANY_ACTION, cmb::NIL, CMB_ANY_OBJECT) == hn ? 1u : 0u;
            counter[5] = cmb_event_pattern_count(USER + 1u, CMB_ANY_SUBJECT, CMB_ANY_OBJECT);
        }
        else if (which == 3u) {
            awaited = cmb_event_schedule(USER, 0u, 0, 5.0, 0);
            cmb_process_start(cmb_process_create(0u, 0, 0u));
            (void)cmb_event_schedule(CLEAR, 0u, 0, 1.0, 0);
        }
        else {
            cmb_event_queue_initialize(2.0);
            counter[0] = (uint64_t)__double_as_longlong(cmb_time());
            counter[1] = sim.status;
            (void)cmb_event_schedule(USER, 0u, 0, 3.0, 0);
            cmb_event_queue_initialize(5.0);
            counter[2] = (uint64_t)__double_as_longlong(cmb_time());
        }
    }

    CMB_FN void finish(S &, cmb::TrialOut &out)
    {
        out.objects = 0u;
        out.sum_wait = 0.0;
        out.max_queue = 0u;
        for (int k = 0; k < 8; k++) out.counters[k] = counter[k];
    }
};

// ---------------------------------------------------------------- running trials
struct HostResult {
    uint64_t events, objects;
    double   t_end, sum_wait;
    uint64_t max_fel, max_queue;
    uint64_t counter[8];
    uint32_t status, pad;
};

static const ZigHot &hot_tables()
{
    static ZigHot hot;
    static bool ready = false;
    if (!ready) {
        for (int i = 0; i < 256; i++) {
            hot.exp_x[i] = zig::zig_exp_x[i];
            hot.nor_x[i] = zig::zig_nor_x[i];
        }
        ready = true;
    }
    return hot;
}

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
static void run_general(uint64_t seed, const cmb::TrialIn &in, HostResult &r, uint64_t trace_cap, uint64_t *tk, double *tt)
{
    static std::vector<unsigned char> mem(1u << 20);
    unsigned long long cursor = 0;
    cmb::Arena arena{mem.data(), &cursor, mem.size()};
    cmb::Sim sim;
    ModelT<cmb::Sim> m;
    cmb::TrialOut o;
    sim.init(seed, &hot_tables(), arena);
    if (trace_cap) cmb::run_one_trial<ModelT<cmb::Sim>, true>(sim, m, in, o, trace_cap, tk, tt);
    else           cmb::run_one_trial<ModelT<cmb::Sim>, false>(sim, m, in, o, 0u, nullptr, nullptr);
    copy_out(sim, o, r);
}

// NPROC, NEVENT: the static tier's sim as the model's library builds it (cmb::StaticSimOf)
template <template <class> class ModelT, int NPROC, int NEVENT>
static void run_static(uint64_t seed, const cmb::TrialIn &in, HostResult &r, uint64_t trace_cap, uint64_t *tk, double *tt)
{
    using S = cmb::StaticSimOf<ModelT, NPROC, 0, NEVENT>;
    static_assert(S::WAITS, "the tier's second form with events by handle");
    S sim;
    ModelT<S> m;
    cmb::TrialOut o;
    double win[cmb::STATIC_WINDOW];
    sim.init(seed, &hot_tables(), win, 1u, nullptr, 0u);
    cmb::static_run_trial_host(sim, m, in, o, trace_cap, tk, tt);
    copy_out(sim, o, r);
}

extern "C" {

uint32_t host_event_any_subject(void) { return CMB_ANY_SUBJECT; }

// EventTestT at `seed` (the generator's seed itself, as test_event -s takes it).  engine 0: the general engine, printing the
// reference's text into out (cap bytes, NUL-terminated).  engine 1: the static tier first - *flag_point = the first of its dumps
// at which the trial was flagged (99 = never), status = its status - then, if it was flagged, the general engine again from the
// same template, printing, as the library's launch re-runs it.  Returns the status of the static run (engine 1) or of the run.
uint32_t host_event_test_text(int engine, uint64_t seed, char *out, uint64_t cap, uint32_t *flag_point)
{
    cmb::TrialIn in{};
    HostResult r{};
    uint32_t status = 0u;
    g_flag_point = 99u;
    if (engine == 1) {
        run_static<EventTestFlagged, 1, EVENT_TEST_SLOTS>(seed, in, r, 0u, nullptr, nullptr);
        status = r.status;
        if (flag_point) *flag_point = g_flag_point;
        if ((status & (TRIAL_ERR_PROC_OVERFLOW | TRIAL_ERR_FEL_OVERFLOW)) == 0u) {
            if (out && cap) out[0] = '\0';
            return status;
        }
    }
    g_text.clear();
    say("Using seed: 0x%" PRIx64 "\n", seed);
    run_general<EventTestPrinted>(seed, in, r, 0u, nullptr, nullptr);
    line_of('-');
    g_text += "--------------------- Event queue ---------------------\n-------------------------------------------------------\n";
    line_of('*');
    if (engine != 1) status = r.status;
    if (out && cap) {
        std::strncpy(out, g_text.c_str(), cap - 1u);
        out[cap - 1u] = '\0';
    }
    return status;
}

// model 0 = EventTestT, 1 = EventChurnT, 2 = EdgeT (case = params0); engine 0 = the general engine, 1 = the static tier (no re-run:
// its own row and status).  Trial i is seeded fmix64(master, first + i).  Returns 0, -1 for another model or engine.
int host_event_run_trials(int model, int engine, uint64_t master, uint64_t first, uint64_t count, uint64_t num_objects,
                          double srv_mean, double params0, uint64_t trace_cap, uint64_t *trace_key, double *trace_time,
                          HostResult *out)
{
    if (model < 0 || model > 2 || engine < 0 || engine > 1) return -1;
    for (uint64_t i = 0; i < count; i++) {
        cmb::TrialIn in{};
        in.arr_mean = 1.0;
        in.srv_mean = srv_mean;
        in.num_objects = num_objects;
        in.num_params = 1u;
        in.params[0] = params0;
        in.trial = first + i;
        const uint64_t seed = fmix64(master, first + i);
        uint64_t *tk = trace_cap ? trace_key + i * trace_cap : nullptr;
        double *tt = trace_cap ? trace_time + i * trace_cap : nullptr;
        if (model == 0) {
            if (engine == 0) run_general<EventTest>(seed, in, out[i], trace_cap, tk, tt);
            else             run_static<EventTest, 1, EVENT_TEST_SLOTS>(seed, in, out[i], trace_cap, tk, tt);
        }
        else if (model == 1) {
            if (engine == 0) run_general<EventChurnT>(seed, in, out[i], trace_cap, tk, tt);
            else             run_static<EventChurnT, 3, EVENT_CHURN_SLOTS>(seed, in, out[i], trace_cap, tk, tt);
        }
        else {
            if (engine == 0) run_general<EdgeT>(seed, in, out[i], trace_cap, tk, tt);
            else             run_static<EdgeT, 2, 4>(seed, in, out[i], trace_cap, tk, tt);
        }
    }
    return 0;
}

}  // extern "C"
