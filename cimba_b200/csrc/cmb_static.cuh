// cmb_static.cuh - the static tier of the authoring surface.
//
// The general engine (cmb_device.cuh) runs ANY model, and pays for it: every container is in memory and grows.  Many models
// need none of that: a FIXED set of processes that only hold and wait at queues - the benchmark's M/M/1
// (benchmark/MM1_multi.c:52-125), G/G/1, a tandem line.  For those, the same model text - the same CMB_PROCESS_* /
// CMB_OBJECTQUEUE_* macros, the same cmb_* names - compiles against cmb::StaticSim<NPROC, NQUEUE, NEVENT> instead of cmb::Sim:
//   * the event list is one slot per process in registers (SlotFel, engine.cuh): a process that can only hold or wait owns at
//     most one pending event, so an insert is a register write and pop-min an NPROC-way compare;
//   * process records, guards (a bit and a sequence number per process) and the model struct stay in registers: process ids
//     are compile-time constants after inlining, nothing takes an address;
//   * a queue is a ring with its oldest 32 entries in shared memory and the rest in an HBM ring (StampRing, engine.cuh); a
//     cmb_buffer is two counters; a cmb_resourcepool is two counters and a holding per process, a cmb_resource its holder;
//     each can keep its time-weighted history (S::recorded_queue_type, ..._buffer_type, ..._resourcepool_type, ..._resource_type);
//   * blocking calls are commands carried out by the dispatcher where the warp is together, and the ziggurat's slow path
//     is taken by parked lanes in batches - as in the fused kernels (queue_model.cuh, whose shape this generalises); a hold
//     of any distribution can be drawn there too (CMB_PROCESS_HOLD_SAMPLED: rectangles first, rewind + park + batch otherwise).
//   * every cmb_random_* distribution, cmb_random_alias_* and cmb_datasummary_* / cmb_wtdsummary_* (cmb_device.cuh, bottom) inline
//     here (inline_draws below): no call takes the generator's address, and in a sampler each of them - rejection loops included -
//     gives up when a ziggurat draw leaves the rectangles (distributions.cuh), so CMB_PROCESS_HOLD_SAMPLED takes any of them.
// A model that says `static constexpr bool static_interrupts = true;` gets the tier's second form (StaticSim<..., PRE = true>):
// process priorities (cmb_process_create with a priority, cmb_process_priority_set), cmb_process_interrupt, CMB_RESOURCEPOOL_PREEMPT
// and CMB_RESOURCE_PREEMPT, and - with a `static_holdables` hook naming its pools and resources - a process stopped or exiting
// while it holds from one of them.  Its guards are then literal binary heaps in the reference's layout (the wait-list order is
// not a strict weak order, SURVEY.md quirk 1, so the physical heap decides who is woken), its interrupts and pre-emptions take
// the model's NEVENT spare event slots, and cmb_random_flip has its per-trial cache.
// In either form a cmb_priorityqueue (S::priorityqueue_type, S::recorded_priorityqueue_type) is a table of STATIC_PQ_CAP objects
// scanned under its strict order, and a cmb_condition (S::condition_type) a literal heap of waiters with their predicates, whose
// wake-ups take the waiters' own event slots; a model that reports cmb::Sim's fel_high says `static constexpr bool
// static_fel_high = true;` (StaticSimHigh).
// A second-form model that also says `static constexpr bool static_waits = true;` (StaticSim<..., PRE = true, W = true>) has
// cmb_process_timer_add / _timer_cancel / _timers_clear / _timer_set, cmb_process_resume and CMB_PROCESS_YIELD,
// CMB_PROCESS_WAIT_PROCESS and CMB_PROCESS_WAIT_EVENT, cmb_event_cancel / _reschedule / _reprioritize / _is_scheduled / _time /
// _priority and cmb_event_pattern_find / _count / _cancel on its own events, and cmb_resourceguard_register with a condition's guard observing another guard: timers, resumes and wake-ups take
// spare slots, and each process has one wait record.
// What the tier does NOT have - process creation beyond NPROC; without static_interrupts priorities other than 0, interrupts and
// pre-emption, and without static_waits timers, resumes, waits on processes and events, events by handle and observers; a process
// that ends while it holds from two or more containers, or from any without the hook; a queue that outgrows window + ring or its
// table, a spare slot or a guard heap too few; a cancel of an event somebody waits on by timers_clear, cancel_awaiteds or a stop
// (whose wake-up order the tier does not keep), a second wait while one is registered, a pattern find with two or more matches or a
// pattern cancel of two or more events with waiters (both decided by the general engine's heap-array order) - is not an error: the trial is flagged and
// the launch re-runs it on the general engine from the SAME model template (launch_static_model below), so the answer is the
// reference's either way.
//
// A model is `template <class S> struct M` with S = cmb::Sim or cmb::StaticSim<...>, its queues declared as
// `typename S::queue_type`, exported with CMB_EXPORT_STATIC_MODEL(M, NPROC, NQUEUE, "name") (or ..._EVENTS(M, NPROC, NQUEUE,
// NEVENT, "name")).  In this library: mm1_model.cuh, gg1_model.cuh, mm1_recorded_model.cuh, tutorial1_model.cuh (the reference's
// first tutorial: two processes, a buffer, three events); with static_interrupts, workshop_model.cuh's ToolT (test/test_resource.c)
// and WorkshopT (test/test_buffer.c and the buffer-and-resource world: the buffer in the second form), cheese_model.cuh
// (test/test_resourcepool.c), coverage_models.cuh's PoolFightT (test/test_resourcepool.c's cast with checks) and
// tutorial2_model.cuh (tutorial/tut_2_1.c), and with priority queues and conditions guarded_model.cuh (test/test_objectqueue.c,
// test/test_priorityqueue.c) and coverage_models.cuh's QueueAndTideT; with static_waits coverage_models.cuh's FrontDeskT;
// examples/tandem_model.cuh; examples/clinic_model.cuh (every cmb_random distribution, alias tables, summaries); with static_waits
// examples/event_model.cuh (the event list's queries, clear and patterns).
#pragma once

#include <type_traits>

#include "cmb_kernel.cuh"

namespace cimba_b200 {
namespace cmb {

constexpr int STATIC_WINDOW = 32;       // on-chip entries per queue and trial
constexpr int STATIC_BLOCK = 64;

// One event slot per process (the shape of SlotFel, engine.cuh), the action packed into the key's two low bits as mm1_fast.cuh
// does: key = (issue counter << 2) | action, 0 = empty.  Counters are unique, so ordering by this word is ordering by issue
// counter - the reference's tie-break (src/cmi_hashheap.c:55-80).
template <int N, bool PRIO = false>
struct StaticFel {
    double   t[N];
    uint32_t key[N];
    int32_t  prio[N];           // PRIO only (a model with events of its own): higher goes first at equal times
    uint32_t issued;

    CMB_FN void clear()
    {
#pragma unroll
        for (int i = 0; i < N; i++) {
            t[i] = __longlong_as_double(0x7ff0000000000000LL);
            key[i] = 0u;
            prio[i] = 0;
        }
        issued = 0u;
    }

    CMB_FN bool schedule(int p, uint32_t action, double time, int32_t priority = 0)     // false: slot p already had a pending event
    {
        const uint32_t k = (++issued << 2) | action;
        bool ok = true;
#pragma unroll
        for (int i = 0; i < N; i++) {
            if (i == p) {
                ok = key[i] == 0u;
                t[i] = time;
                key[i] = k;
                if (PRIO) prio[i] = priority;
            }
        }
        return ok;
    }

    CMB_FN void drop(int p)
    {
#pragma unroll
        for (int i = 0; i < N; i++) {
            if (i == p) {
                t[i] = __longlong_as_double(0x7ff0000000000000LL);
                key[i] = 0u;
            }
        }
    }

    // cmi_hashheap_dequeue: the first entry under (time asc, priority desc, key asc) - default_compare, src/cmi_hashheap.c:55-80;
    // false when the list is empty
    CMB_FN bool pop(int &p, uint32_t &action, double &time, uint32_t &counter)
    {
        int best = 0;
        double bt = t[0];
        uint32_t bk = key[0];
        int32_t bp = PRIO ? prio[0] : 0;
#pragma unroll
        for (int i = 1; i < N; i++) {
            bool before;
            if (PRIO) {
                before = (t[i] < bt) | ((t[i] == bt) & ((prio[i] > bp) | ((prio[i] == bp) & (key[i] < bk))));
            }
            else {
                before = (t[i] < bt) | ((t[i] == bt) & (key[i] < bk));
            }
            if (before) {
                best = i;
                bt = t[i];
                bk = key[i];
                if (PRIO) bp = prio[i];
            }
        }
        drop(best);
        p = best;
        action = bk & 3u;
        time = bt;
        counter = bk >> 2;
        return bk != 0u;
    }
};

// the wait list of a guard whose only possible waiters are the NPROC processes: who waits, and since when (FIFO)
template <int NPROC>
struct static_guard {
    uint32_t waiting;
    uint32_t seq[NPROC];

    CMB_FN void reset()
    {
        waiting = 0u;
#pragma unroll
        for (int i = 0; i < NPROC; i++) seq[i] = 0u;
    }
};

// ... and the same wait list where waiters have priorities (StaticSim<..., PRE = true>): cmb::HashHeap<GuardOrder>'s heap with
// its physical layout - 1-based, the same sift and remove steps (src/cmi_hashheap.c:277-370, 486-579) - because guard_queue_check
// is not a strict weak order (SURVEY.md quirk 1) and the layout decides who is at the top.  At most NPROC entries: a stopped
// process's entry stays (quirk 2), so only a process restarted while its old entry waits can overflow it (the trial is flagged).
// Entries are found by key with a scan.
struct static_guard_entry {
    double   d;                 // when the process began to wait
    uint32_t key;               // the guard sequence number it waits under
    int32_t  prio;              // its priority then
    uint32_t subj;
};

// a cmb_condition's waiter also carries its predicate: m.demand(sim, demand, subj, ctx)
struct static_condition_entry : static_guard_entry {
    uint32_t demand;
    int32_t  ctx;
};

template <int NPROC, class E = static_guard_entry>
struct static_heap_guard {
    using Entry = E;
    uint32_t count;
    Entry    e[NPROC + 1];

    CMB_FN void reset() { count = 0u; }

    static CMB_FN bool before(const Entry &a, const Entry &b)          // GuardOrder, cmb_device.cuh
    {
        if (a.prio > b.prio) return true;
        if (a.d < b.d) return true;
        if (a.key < b.key) return true;
        return false;
    }

    CMB_FN void sift_up(uint32_t k)                                    // heap_up
    {
        const Entry moving = e[k];
        uint32_t parent;
        while ((parent = (k >> 1)) > 0u) {
            if (!before(moving, e[parent])) break;
            e[k] = e[parent];
            k = parent;
        }
        e[k] = moving;
    }

    CMB_FN void sift_down(uint32_t k)                                  // heap_down
    {
        const Entry moving = e[k];
        const uint32_t last_parent = count >> 1;
        while (k <= last_parent) {
            uint32_t child = k << 1;
            if (child + 1u <= count && before(e[child + 1u], e[child])) child++;
            if (before(moving, e[child])) break;
            e[k] = e[child];
            k = child;
        }
        e[k] = moving;
    }

    CMB_FN bool push(double d, uint32_t key, int32_t prio, uint32_t subj)   // cmi_hashheap_enqueue; false = full
    {
        if (count >= (uint32_t)NPROC) return false;
        const uint32_t at = ++count;
        e[at].d = d;
        e[at].key = key;
        e[at].prio = prio;
        e[at].subj = subj;
        sift_up(at);
        return true;
    }

    CMB_FN bool push(const Entry &x)                                   // ... an entry with more than those four fields
    {
        if (count >= (uint32_t)NPROC) return false;
        const uint32_t at = ++count;
        e[at] = x;
        sift_up(at);
        return true;
    }

    CMB_FN void pop()                                                  // cmi_hashheap_dequeue (the top entry leaves)
    {
        if (count > 1u) {
            e[1] = e[count];
            count--;
            if (count > 1u) sift_down(1u);
        }
        else {
            count = 0u;
        }
    }

    CMB_FN void remove(uint32_t key)                                   // cmi_hashheap_remove
    {
        uint32_t at = 0u;
        for (uint32_t k = 1u; k <= count; k++) {
            if (at == 0u && e[k].key == key) at = k;
        }
        if (at == 0u) return;
        if (at == count) {
            count--;
            return;
        }
        const bool down = before(e[at], e[count]);
        e[at] = e[count];
        count--;
        if (down) sift_down(at);
        else sift_up(at);
    }
};

template <int NPROC, bool PRE>
using static_guard_of = typename std::conditional<PRE, static_heap_guard<NPROC>, static_guard<NPROC>>::type;

// RECORD: the queue can keep its length history (cmb_objectqueue_recording_start, src/cmb_objectqueue.c:161-177), folded on the
// fly into the time-weighted summary cmb_timeseries_summarize would make of it (TimeWeighted, summary.cuh).  A queue type of its
// own (S::recorded_queue_type) so that models that never record carry neither the registers nor the sampling code.  C is the
// container, whose recorded_level() the history follows.  The level and the clock are read only where the reference reads them -
// after the recording flag is tested, after the history is reset - so that a model whose containers live in local memory loads
// nothing earlier than it must.
template <bool RECORD, class C>
struct static_history {
    template <class S> CMB_FN void start(const S &) {}
    template <class S> CMB_FN void stop(const S &) {}
    template <class S> CMB_FN void sample(const S &) {}
};
template <class C>
struct static_history<true, C> {
    uint32_t recording;
    TimeWeighted history;

    template <class S>
    CMB_FN void start(const S &sim)                 // cmb_*_recording_start
    {
        recording = 1u;
        history.start();
        history.sample(static_cast<const C *>(this)->recorded_level(), sim.now);
    }

    template <class S>
    CMB_FN void stop(const S &sim)                  // cmb_*_recording_stop
    {
        sample(sim);
        recording = 0u;
    }

    template <class S>
    CMB_FN void sample(const S &sim)                // record_sample: the level changed
    {
        if (recording) history.sample(static_cast<const C *>(this)->recorded_level(), sim.now);
    }
};

template <int NPROC, bool RECORD = false, bool PRE = false>
struct static_objectqueue : static_history<RECORD, static_objectqueue<NPROC, RECORD, PRE>> {
    static_guard_of<NPROC, PRE> front, rear;
    StampRing<STATIC_WINDOW> ring;
    uint64_t capacity;
    uint32_t longest;
    uint32_t length;            // = ring.len (cmb_objectqueue_length)

    CMB_FN double recorded_level() const { return (double)ring.len; }
};

// struct cmb_buffer for a fixed set of processes (amounts put and got in parts, src/cmb_buffer.c:194-346)
template <int NPROC, bool RECORD = false, bool PRE = false>
struct static_buffer : static_history<RECORD, static_buffer<NPROC, RECORD, PRE>> {
    static_guard_of<NPROC, PRE> front, rear;
    uint64_t level, capacity;

    CMB_FN double recorded_level() const { return (double)level; }
};

// struct cmb_resourcepool for a fixed set of processes (src/cmb_resourcepool.c): the holders' records are a bit and an amount
// per process, in registers like the rest (a holder's priority is its process's: cmb_process_priority_set moves both); the
// history, when kept, is of in_use
template <int NPROC, bool RECORD = false, bool PRE = false>
struct static_resourcepool : static_history<RECORD, static_resourcepool<NPROC, RECORD, PRE>> {
    static_guard_of<NPROC, PRE> guard;
    uint64_t capacity, in_use;
    uint32_t holding;           // bit i: process i has a holder record (cmb_resourcepool_held_by_process finds it)
    uint64_t held[NPROC];       // ... and the amount it holds

    CMB_FN double recorded_level() const { return (double)in_use; }
};

// struct cmb_resource, the binary semaphore (src/cmb_resource.c); the history, when kept, is 1 while held, 0 while free
template <int NPROC, bool RECORD = false, bool PRE = false>
struct static_resource : static_history<RECORD, static_resource<NPROC, RECORD, PRE>> {
    static_guard_of<NPROC, PRE> guard;
    uint32_t holder;            // process index, NIL = free

    CMB_FN double recorded_level() const { return holder != NIL ? 1.0 : 0.0; }
};

// struct cmb_priorityqueue (src/cmb_priorityqueue.c) for a fixed set of processes: at most STATIC_PQ_CAP objects, in a table
// in the thread's local memory like the guard heaps.  Its order (PrioOrder: priority descending, then handle ascending) is a
// strict total order, so the first entry of the unsorted table under it is exactly the one the reference's heap gives up next,
// and no heap layout needs keeping.  A put that finds the table full while `capacity` has room flags the trial (no HBM spill).
constexpr int STATIC_PQ_CAP = 16;

struct static_pq_entry {
    uint64_t obj;
    uint64_t handle;            // the key cmb_priorityqueue_put hands out: 1, 2, ... per queue (HashHeap::issued)
    int32_t  prio;
};

template <int NPROC, bool RECORD = false, bool PRE = false>
struct static_priorityqueue : static_history<RECORD, static_priorityqueue<NPROC, RECORD, PRE>> {
    static_guard_of<NPROC, PRE> front, rear;
    static_pq_entry e[STATIC_PQ_CAP];
    uint64_t capacity;
    uint64_t issued;
    uint32_t count;

    CMB_FN double recorded_level() const { return (double)count; }
};

// struct cmb_condition (src/cmb_condition.c) for a fixed set of processes: its wait list is always the literal heap, in both
// forms of the tier, because cmb_condition_signal goes over it in array order and that order decides the wake-ups' keys
template <int NPROC>
struct static_condition {
    static_heap_guard<NPROC, static_condition_entry> guard;
};

// What StaticSim<..., PRE = true> keeps besides: each process's priority (cmb_process_priority) and the key of its guard entry
// (cmb_process::guard_key), and cmb_random_flip's cache - per trial, as the general engine has it.  A base class, so that the
// tier's first form (PRE = false) keeps its layout.
template <int NPROC, bool PRE>
struct StaticPriorities {
};
template <int NPROC>
struct StaticPriorities<NPROC, true> {
    int32_t   prio[NPROC];
    uint32_t  gkey[NPROC];
    FlipCache flips;
};

// What StaticSim<..., W = true> keeps besides (a model's static_waits): what each process waits on with CMB_PROCESS_WAIT_PROCESS
// or CMB_PROCESS_WAIT_EVENT - one thing at a time - and since when, and the guards that observe others (cmb_resourceguard_register).
// A base class, so that every other model keeps its layout.
constexpr int STATIC_OBSERVERS = 2;

template <int NPROC, bool W>
struct StaticWaits {
};
template <int NPROC>
struct StaticWaits<NPROC, true> {
    enum : uint32_t { WAIT_NONE = 0u, WAIT_PROCESS = 1u, WAIT_EVENT = 2u };
    uint32_t wkind[NPROC];
    uint32_t wref[NPROC];       // the process index, or the event's handle
    uint32_t wseq[NPROC];       // the order of the waits: the reference's waiter lists are woken latest first
    uint32_t wait_seq;
    uint32_t nobs;
    const void *obs_from[STATIC_OBSERVERS];                                     // the guard observed ...
    static_heap_guard<NPROC, static_condition_entry> *obs_to[STATIC_OBSERVERS]; // ... and the condition's guard that observes it
};

// NEVENT: how many events of its own (cmb_event_schedule) a model may have pending at once; with any, the event list also
// orders by priority.  PRE (the model's static_interrupts): priorities, interrupts and pre-emption, whose events for a process
// besides its own slot's - an interrupt, a resource pre-emption - take spare slots too.  W (the model's static_waits, which needs
// PRE): timers, cmb_process_resume, waits on processes and events, the model's events by handle, and observers - their events in
// spare slots as well.
template <int NPROC, int NQUEUE, int NEVENT = 0, bool PRE = false, bool W = false>
struct StaticSim : StaticPriorities<NPROC, PRE>, StaticWaits<NPROC, W> {
    using queue_type = static_objectqueue<NPROC, false, PRE>;
    using recorded_queue_type = static_objectqueue<NPROC, true, PRE>;
    using buffer_type = static_buffer<NPROC, false, PRE>;
    using recorded_buffer_type = static_buffer<NPROC, true, PRE>;
    using resourcepool_type = static_resourcepool<NPROC, false, PRE>;
    using recorded_resourcepool_type = static_resourcepool<NPROC, true, PRE>;
    using resource_type = static_resource<NPROC, false, PRE>;
    using recorded_resource_type = static_resource<NPROC, true, PRE>;
    using priorityqueue_type = static_priorityqueue<NPROC, false, PRE>;
    using recorded_priorityqueue_type = static_priorityqueue<NPROC, true, PRE>;
    using condition_type = static_condition<NPROC>;
    using guard_type = static_guard_of<NPROC, PRE>;
    using condition_guard = static_heap_guard<NPROC, static_condition_entry>;
    static constexpr int PROCESSES = NPROC;
    static constexpr int QUEUES = NQUEUE;
    static constexpr int SLOTS = NPROC + NEVENT;
    static constexpr bool INTERRUPTS = PRE;
    static constexpr bool WAITS = W;
    static constexpr bool inline_draws = true;      // every cmb_random_* inlines and honours hot_only (distributions.cuh)
    static_assert(NPROC >= 1 && NPROC <= 32, "a guard's wait list is a 32-bit mask of processes");
    static_assert(!PRE || NEVENT > 0, "interrupts and pre-emptions take spare event slots, and the event list must order by priority");
    static_assert(!W || PRE, "timers, resumes and waits on processes and events need the tier's second form (static_interrupts)");
    static constexpr uint32_t HOLD_BITS = NPROC <= 8 ? 4u : (NPROC <= 16 ? 2u : 1u);
    static constexpr uint32_t HOLD_MAX = (1u << HOLD_BITS) - 1u;
    struct Proc {
        uint32_t pc, status, kind, ctx;
        double   f[2];
        uint64_t u[2];
        uint64_t fr[3];         // scratch of the blocking calls in progress (a buffer call's remaining / obtained amounts)
        int64_t  exit_value;
    };
    struct UserEvent {
        uint32_t act, subj;
        int64_t  arg;
    };
    Sfc64          rng;
    const ZigHot  *hot;
    double         now;
    uint32_t       status;
    uint32_t       current;
    uint32_t       current_event;
    uint32_t       pops;
    uint32_t       nproc, nqueue, guard_seq;
    // how many pools and resources each process holds from, HOLD_BITS per process.  The reference drops a process's
    // holdings when it exits or is stopped (cmi_process_drop_resources, src/cmb_process.c:507-527); this tier does not, and
    // flags the trial instead.  One word, in what would otherwise be padding: a model that holds nothing keeps its layout.
    uint32_t       holds;
    Proc           proc[NPROC];
    StaticFel<NPROC + NEVENT, (NEVENT > 0)> fel;
    UserEvent      uev[NEVENT > 0 ? NEVENT : 1];
    uint32_t       cmd;
    uint32_t       cmd_sample;
    double         cmd_value;
    int64_t        cmd_exit;
    bool           hot_only;        // a sampler is being tried with the ziggurats' rectangles only ...
    bool           hot_failed;      // ... and that was not enough: the draw will be repeated with the slow paths, in a batch
    // where this trial's queues live: column `tid` of the CTA's shared-memory rings, and its HBM rings
    double        *ring_win;
    uint32_t       ring_stride;
    double        *spill;
    uint32_t       spill_cap;

    CMB_FN void init(uint64_t seed, const ZigHot *tables, double *win, uint32_t stride, double *spill_rings, uint32_t cap)
    {
        rng.seed(seed);
        hot = tables;
        now = 0.0;
        status = 0u;
        current = NIL;
        current_event = 0u;
        pops = 0u;
        nproc = nqueue = guard_seq = 0u;
        holds = 0u;
        fel.clear();
        cmd = CMD_NONE;
        cmd_sample = 0u;
        cmd_value = 0.0;
        cmd_exit = 0;
        hot_only = hot_failed = false;
        ring_win = win;
        ring_stride = stride;
        spill = spill_rings;
        spill_cap = cap;
#pragma unroll
        for (int i = 0; i < NPROC; i++) {
            proc[i].pc = 0u;
            proc[i].status = PROC_CREATED;
            proc[i].kind = 0u;
            proc[i].ctx = 0u;
            proc[i].f[0] = proc[i].f[1] = 0.0;
            proc[i].u[0] = proc[i].u[1] = 0u;
            proc[i].fr[0] = proc[i].fr[1] = proc[i].fr[2] = 0u;
            proc[i].exit_value = 0;
        }
        if constexpr (PRE) {
#pragma unroll
            for (int i = 0; i < NPROC; i++) {
                this->prio[i] = 0;
                this->gkey[i] = 0u;
            }
            this->flips.bits = 0u;
            this->flips.pos = 0u;
        }
        if constexpr (W) {
#pragma unroll
            for (int i = 0; i < NPROC; i++) {
                this->wkind[i] = this->WAIT_NONE;
                this->wref[i] = 0u;
                this->wseq[i] = 0u;
            }
            this->wait_seq = 0u;
            this->nobs = 0u;
        }
    }

    // f(i) for the process i == pid.  Unrolled, so that i is a compile-time constant in every copy of f and the per-process
    // records it touches (proc[i], prio[i], a guard's seq[i], ...) stay in registers; f must not let an address of them escape.
    template <class F>
    static CMB_FN void at_process(uint32_t pid, F &&f)
    {
#pragma unroll
        for (int i = 0; i < NPROC; i++) {
            if ((uint32_t)i == pid) f(i);
        }
    }

    // the priority of process pid (0 in the tier's first form, which has none)
    CMB_FN int32_t prio_of(uint32_t pid) const
    {
        int32_t p = 0;
        if constexpr (PRE) at_process(pid, [&](int i) { p = this->prio[i]; });
        return p;
    }

    CMB_FN uint32_t holds_of(uint32_t pid) const { return (holds >> (pid * HOLD_BITS)) & HOLD_MAX; }

    // process pid began (+1) or ceased (-1) to hold from a pool or a resource.  More holdings at once than HOLD_BITS count:
    // the trial goes to the general engine.
    CMB_FN void holds_add(uint32_t pid, int32_t d)
    {
        const uint32_t c = holds_of(pid);
        if (d > 0) {
            if (c == HOLD_MAX) status |= TRIAL_ERR_PROC_OVERFLOW;
            else holds += 1u << (pid * HOLD_BITS);
        }
        else if (c > 0u) {
            holds -= 1u << (pid * HOLD_BITS);
        }
    }

    // cmb_event_schedule(action, subject, object, time, priority) for an event of the model's own (src/cmb_event.c:123-140):
    // one of the NEVENT spare slots.  Returns the handle (= key), 0 if there is no slot left (the trial is flagged).
    CMB_FN uint64_t schedule(uint32_t act, uint32_t subj, int64_t arg, double t, int64_t prio)
    {
        int slot = -1;
#pragma unroll
        for (int i = NPROC; i < NPROC + NEVENT; i++) {
            if (slot < 0 && fel.key[i] == 0u) slot = i;
        }
        if (slot < 0) {
            status |= TRIAL_ERR_FEL_OVERFLOW;
            return 0u;
        }
        (void)fel.schedule(slot, 0u, t, (int32_t)prio);
#pragma unroll
        for (int i = 0; i < NEVENT; i++) {
            if (i == slot - NPROC) {
                uev[i].act = act;
                uev[i].subj = subj;
                uev[i].arg = arg;
            }
        }
        return (uint64_t)fel.issued;
    }

    // cmb_process_create + cmb_process_initialize.  One process more than the tier holds, or a priority without PRE: the
    // trial goes to the general engine.
    CMB_FN uint32_t process_create(uint32_t kind, int64_t prio, uint32_t ctx)
    {
        const uint32_t id = nproc;
        if (id >= (uint32_t)NPROC || (!PRE && prio != 0)) {
            status |= TRIAL_ERR_PROC_OVERFLOW;
            return 0u;
        }
        nproc = id + 1u;
        at_process(id, [&](int i) {
            proc[i].kind = kind;
            proc[i].ctx = ctx;
            proc[i].status = PROC_CREATED;
            if constexpr (PRE) this->prio[i] = (int32_t)prio;
        });
        return id;
    }

    CMB_FN void process_start(uint32_t pid)             // src/cmb_process.c:127-135
    {
        if (!fel.schedule((int)pid, ACT_START, now, prio_of(pid))) status |= TRIAL_ERR_FEL_OVERFLOW;
        if (holds_of(pid) != 0u) status |= TRIAL_ERR_PROC_OVERFLOW;    // restarted after it ended holding: see static_trial_end
    }

    // cmb_process_hold after its yield (src/cmb_process.c:274-284): woken by anything but its own wake-up, the process drops
    // that (pending in its slot, if an interrupt did not take it already)
    CMB_FN int64_t hold_end(uint32_t pid, int64_t sig)
    {
        if constexpr (PRE) {
            if (sig != CMB_PROCESS_SUCCESS) fel.drop((int)pid);
        }
        return sig;
    }

    // cmi_process_cancel_awaiteds + cmb_event_pattern_cancel(ANY, pid, ANY) (src/cmb_process.c:581-620, as cmb::Sim does it):
    // the process's slot, and every spare-slot event of the engine's own (act < ACT_CMB_USER) about it.  Its guard entry stays
    // (SURVEY.md quirk 2).  Nothing is rescheduled, so no key is issued and the order of the drops does not matter.  W: its wait on
    // a process or an event ends too (:529-551, src/cmb_event.c:486-508); an event cancelled here that others wait on would wake
    // them with keys in the order of the general engine's heap array, which the tier does not keep, so the trial is flagged.
    CMB_FN void cancel_awaiteds(uint32_t pid)
    {
        fel.drop((int)pid);
#pragma unroll
        for (int i = 0; i < NEVENT; i++) {
            if (fel.key[NPROC + i] != 0u && uev[i].act < ACT_CMB_USER && uev[i].subj == pid) {
                if constexpr (W) {
                    if (has_waiters(fel.key[NPROC + i] >> 2)) status |= TRIAL_ERR_PROC_OVERFLOW;
                }
                fel.drop(NPROC + i);
            }
        }
        if constexpr (W) wait_clear(pid);
    }

    // cmb_process_interrupt (:653-666): an event at `now` in a spare slot; without PRE, the general engine's business
    CMB_FN void interrupt(uint32_t pid, int64_t sig, int64_t pri)
    {
        if constexpr (PRE) (void)schedule(ACT_CMB_WAKE_INTERRUPT, pid, sig, now, pri);
        else status |= TRIAL_ERR_PROC_OVERFLOW;
    }

    // ---- W: timers, resume, waits on processes and events, the model's events by handle.  Without W each of these sends the
    // trial to the general engine, so that one model text still compiles for every form.
    // the spare slot of the pending event with this handle (= its key >> 2, what schedule returns), -1 if there is none
    CMB_FN int slot_of(uint64_t handle) const
    {
        int slot = -1;
#pragma unroll
        for (int i = NPROC; i < NPROC + NEVENT; i++) {
            if (fel.key[i] != 0u && (uint64_t)(fel.key[i] >> 2) == handle) slot = i;
        }
        return slot;
    }

    CMB_FN bool has_waiters(uint32_t handle) const
    {
        bool any = false;
        if constexpr (W) {
#pragma unroll
            for (int i = 0; i < NPROC; i++) any |= this->wkind[i] == this->WAIT_EVENT && this->wref[i] == handle;
        }
        return any;
    }

    CMB_FN void wait_clear(uint32_t pid)
    {
        if constexpr (W) at_process(pid, [&](int i) { this->wkind[i] = this->WAIT_NONE; });
    }

    // pid begins to wait on `ref`.  The general engine keeps a list per process; one wait at a time is all a record holds, so a
    // process that begins a second wait while the first is still registered (resumed by a timer, say) goes to the general engine.
    CMB_FN void wait_begin(uint32_t pid, uint32_t kind, uint32_t ref)
    {
        if constexpr (W) {
            const uint32_t s = ++this->wait_seq;
            at_process(pid, [&](int i) {
                if (this->wkind[i] != this->WAIT_NONE) status |= TRIAL_ERR_PROC_OVERFLOW;
                this->wkind[i] = kind;
                this->wref[i] = ref;
                this->wseq[i] = s;
            });
        }
    }

    // every process waiting on (kind, ref), latest first as the reference's lists are walked (wake_process_waiters, src/cmb_process.c:
    // 485-505; wake_event_waiters, src/cmb_event.c:200-221): a wake-up at `now` and the process's priority, one key each
    CMB_FN void wake_waiters(uint32_t kind, uint32_t ref, uint32_t act, int64_t sig)
    {
        if constexpr (W) {
            for (int n = 0; n < NPROC; n++) {
                int who = -1;
                uint32_t latest = 0u;
#pragma unroll
                for (int i = 0; i < NPROC; i++) {
                    if (this->wkind[i] == kind && this->wref[i] == ref && (who < 0 || this->wseq[i] > latest)) {
                        who = i;
                        latest = this->wseq[i];
                    }
                }
                if (who < 0) break;
                wait_clear((uint32_t)who);
                (void)schedule(act, (uint32_t)who, sig, now, prio_of((uint32_t)who));
            }
        }
    }

    CMB_FN void wake_process_waiters(uint32_t pid, int64_t sig) { wake_waiters(this->WAIT_PROCESS, pid, ACT_CMB_WAKE_PROCESS, sig); }
    CMB_FN void wake_event_waiters(uint32_t handle, int64_t sig) { wake_waiters(this->WAIT_EVENT, handle, ACT_CMB_WAKE_EVENT, sig); }

    // cmb_process_timer_add (src/cmb_process.c:316-333): an ACT_CMB_WAKE_TIME in a spare slot that resumes the body with `sig`
    CMB_FN uint64_t timer_add(uint32_t pid, double dur, int64_t sig)
    {
        if constexpr (W) return schedule(ACT_CMB_WAKE_TIME, pid, sig, __dadd_rn(now, dur), prio_of(pid));
        status |= TRIAL_ERR_PROC_OVERFLOW;
        return 0u;
    }

    // cmb_process_timers_clear (:354-381): every timer of the process, and its pending hold's wake-up, which the reference keeps in
    // the same list.  The reference cancels them in the order of that list; only waiters on one of them could tell, and then the
    // trial goes to the general engine.
    CMB_FN void timers_clear(uint32_t pid)
    {
        if constexpr (W) {
            at_process(pid, [&](int i) {
                if ((fel.key[i] & 3u) == ACT_WAKE_TIME) fel.drop(i);
            });
#pragma unroll
            for (int i = 0; i < NEVENT; i++) {
                if (fel.key[NPROC + i] != 0u && uev[i].act == ACT_CMB_WAKE_TIME && uev[i].subj == pid) {
                    if (has_waiters(fel.key[NPROC + i] >> 2)) status |= TRIAL_ERR_PROC_OVERFLOW;
                    fel.drop(NPROC + i);
                }
            }
        }
        else {
            status |= TRIAL_ERR_PROC_OVERFLOW;
        }
    }

    CMB_FN bool timer_cancel(uint32_t, uint64_t handle) { return event_cancel(handle); }       // :338-349

    CMB_FN void timer_set(uint32_t pid, double dur, int64_t sig)                                // clear, then add
    {
        timers_clear(pid);
        (void)timer_add(pid, dur, sig);
    }

    // cmb_process_resume (:751-760): an ACT_CMB_RESUME at `now` and the process's priority, which resumes the body whatever it does
    CMB_FN void resume(uint32_t pid, int64_t sig)
    {
        if constexpr (W) (void)schedule(ACT_CMB_RESUME, pid, sig, now, prio_of(pid));
        else status |= TRIAL_ERR_PROC_OVERFLOW;
    }

    // cmb_process_wait_process up to its yield (:428-452); CMB_PROCESS_WAIT_PROCESS has already looked whether `other` finished
    CMB_FN void wait_process_begin(uint32_t pid, uint32_t other)
    {
        if constexpr (W) wait_begin(pid, this->WAIT_PROCESS, other);
        else status |= TRIAL_ERR_PROC_OVERFLOW;
    }

    // cmb_process_wait_event up to its yield (:461-483): an event that is not pending registers nothing, and the body still yields
    CMB_FN void wait_event_begin(uint32_t pid, uint64_t handle)
    {
        if constexpr (W) {
            if (slot_of(handle) >= 0) wait_begin(pid, this->WAIT_EVENT, (uint32_t)handle);
        }
        else {
            status |= TRIAL_ERR_PROC_OVERFLOW;
        }
    }

    // cmb_event_cancel (src/cmb_event.c:285-302): the event leaves, and its waiters are woken with CMB_PROCESS_CANCELLED
    CMB_FN bool event_cancel(uint64_t handle)
    {
        if constexpr (W) {
            const int slot = slot_of(handle);
            if (slot < 0) return false;
            fel.drop(slot);
            wake_event_waiters((uint32_t)handle, CMB_PROCESS_CANCELLED);
            return true;
        }
        status |= TRIAL_ERR_PROC_OVERFLOW;
        return false;
    }

    CMB_FN bool event_is_scheduled(uint64_t handle)                                             // :145-150
    {
        if constexpr (W) return slot_of(handle) >= 0;
        status |= TRIAL_ERR_PROC_OVERFLOW;
        return false;
    }

    // cmb_event_reschedule / cmb_event_reprioritize (:308-344): the event moves and keeps its key
    CMB_FN bool event_reschedule(uint64_t handle, double t)
    {
        if constexpr (W) {
            const int slot = slot_of(handle);
#pragma unroll
            for (int i = NPROC; i < NPROC + NEVENT; i++) {
                if (i == slot) fel.t[i] = t;
            }
            return slot >= 0;
        }
        status |= TRIAL_ERR_PROC_OVERFLOW;
        return false;
    }

    CMB_FN bool event_reprioritize(uint64_t handle, int64_t pri)
    {
        if constexpr (W) {
            const int slot = slot_of(handle);
#pragma unroll
            for (int i = NPROC; i < NPROC + NEVENT; i++) {
                if (i == slot) fel.prio[i] = (int32_t)pri;
            }
            return slot >= 0;
        }
        status |= TRIAL_ERR_PROC_OVERFLOW;
        return false;
    }

    // ---- the event list as a whole (src/cmb_event.c:75-117), as cmb::Sim has it: the clock set before the first schedule, the
    // occupied slots counted, every slot emptied by a clear.  A clear wakes nobody and issues no key; a wait on a dropped event can
    // never end, so its record goes (the general engine keeps a record that no lookup finds any more).
    CMB_FN void queue_initialize(double start)
    {
        if (fel.issued != 0u) status |= TRIAL_ERR_ARGUMENT;
        else now = start;
    }

    CMB_FN uint64_t queue_count() const
    {
        uint64_t n = 0u;
#pragma unroll
        for (int i = 0; i < NPROC + NEVENT; i++) n += fel.key[i] != 0u ? 1u : 0u;
        return n;
    }

    CMB_FN bool queue_is_empty() const { return queue_count() == 0u; }

    CMB_FN void queue_clear()
    {
        const uint32_t issued = fel.issued;
        fel.clear();
        fel.issued = issued;
        if constexpr (W) {
#pragma unroll
            for (int i = 0; i < NPROC; i++) {
                if (this->wkind[i] == this->WAIT_EVENT) this->wkind[i] = this->WAIT_NONE;
            }
        }
    }

    // ---- W: the model's events by handle and by pattern.  cmb_event_time / _priority of a handle that is not pending flag the
    // trial TRIAL_ERR_ARGUMENT and return 0, as on the general engine.
    CMB_FN double event_time(uint64_t handle)
    {
        double t = 0.0;
        if constexpr (W) {
            const int slot = slot_of(handle);
            if (slot < 0) status |= TRIAL_ERR_ARGUMENT;
#pragma unroll
            for (int i = NPROC; i < NPROC + NEVENT; i++) {
                if (i == slot) t = fel.t[i];
            }
        }
        else {
            status |= TRIAL_ERR_PROC_OVERFLOW;
        }
        return t;
    }

    CMB_FN int64_t event_priority(uint64_t handle)
    {
        int64_t p = 0;
        if constexpr (W) {
            const int slot = slot_of(handle);
            if (slot < 0) status |= TRIAL_ERR_ARGUMENT;
#pragma unroll
            for (int i = NPROC; i < NPROC + NEVENT; i++) {
                if (i == slot) p = fel.prio[i];
            }
        }
        else {
            status |= TRIAL_ERR_PROC_OVERFLOW;
        }
        return p;
    }

    // the spare slots whose events match the pattern (event_matches: the model's own events only), a bit per slot, and how many
    CMB_FN uint64_t pattern_slots(uint32_t act, uint32_t subj, int64_t obj, uint64_t &n) const
    {
        static_assert(NEVENT <= 64, "a pattern's matches are a 64-bit mask of spare slots");
        uint64_t hit = 0u;
        n = 0u;
#pragma unroll
        for (int i = 0; i < NEVENT; i++) {
            if (fel.key[NPROC + i] != 0u && event_matches(uev[i].act, uev[i].subj, uev[i].arg, act, subj, obj)) {
                hit |= 1ull << i;
                n++;
            }
        }
        return hit;
    }

    // cmb_event_pattern_count: the matches, in any order
    CMB_FN uint64_t pattern_count(uint32_t act, uint32_t subj, int64_t obj)
    {
        uint64_t n = 0u;
        if constexpr (W) (void)pattern_slots(act, subj, obj, n);
        else status |= TRIAL_ERR_PROC_OVERFLOW;
        return n;
    }

    // cmb_event_pattern_find: the general engine returns the first match in its heap array, whose order the tier does not keep -
    // exact with at most one match; with two or more the trial is flagged
    CMB_FN uint64_t pattern_find(uint32_t act, uint32_t subj, int64_t obj)
    {
        uint64_t handle = 0u;
        if constexpr (W) {
            uint64_t n;
            const uint64_t hit = pattern_slots(act, subj, obj, n);
            if (n > 1u) status |= TRIAL_ERR_PROC_OVERFLOW;
#pragma unroll
            for (int i = 0; i < NEVENT; i++) {
                if (handle == 0u && ((hit >> i) & 1u) != 0u) handle = fel.key[NPROC + i] >> 2;
            }
        }
        else {
            status |= TRIAL_ERR_PROC_OVERFLOW;
        }
        return handle;
    }

    // cmb_event_pattern_cancel: every match leaves, and its waiters are woken with CMB_PROCESS_CANCELLED.  The general engine
    // cancels in heap-array order, so the keys of the wake-ups are exact here only while at most one of the matches has waiters;
    // with two or more the trial is flagged.
    CMB_FN uint64_t pattern_cancel(uint32_t act, uint32_t subj, int64_t obj)
    {
        if constexpr (W) {
            uint64_t n;
            const uint64_t hit = pattern_slots(act, subj, obj, n);
            int waited = 0;
#pragma unroll
            for (int i = 0; i < NEVENT; i++) {
                if (((hit >> i) & 1u) != 0u && has_waiters(fel.key[NPROC + i] >> 2)) waited++;
            }
            if (waited > 1) status |= TRIAL_ERR_PROC_OVERFLOW;
#pragma unroll
            for (int i = 0; i < NEVENT; i++) {
                if (((hit >> i) & 1u) != 0u) (void)event_cancel(fel.key[NPROC + i] >> 2);
            }
            return n;
        }
        status |= TRIAL_ERR_PROC_OVERFLOW;
        return 0u;
    }

    // cmb_resourceguard_wait up to its yield (src/cmb_resourceguard.c:125-152)
    CMB_FN void guard_wait_cmd(static_guard<NPROC> &g, uint32_t pid, uint32_t, int32_t)
    {
        const uint32_t s = ++guard_seq;
        g.waiting |= 1u << pid;
        at_process(pid, [&](int i) { g.seq[i] = s; });
        cmd = CMD_NONE;
    }

    CMB_FN int64_t guard_wait_end(static_guard<NPROC> &, uint32_t, int64_t sig) { return sig; }

    // cmb_resourceguard_signal (:202-226): the HEAD waiter, if its demand holds - `ok`, which the caller knows (every waiter
    // of a queue's front guard wants content, of its rear guard space)
    CMB_FN void guard_signal(static_guard<NPROC> &g, bool ok)
    {
        if (g.waiting == 0u || !ok) return;
        uint32_t head = 0u, best = 0xffffffffu;
#pragma unroll
        for (int i = 0; i < NPROC; i++) {
            const bool here = ((g.waiting >> i) & 1u) != 0u && g.seq[i] < best;
            if (here) {
                head = (uint32_t)i;
                best = g.seq[i];
            }
        }
        g.waiting &= ~(1u << head);
        if (!fel.schedule((int)head, ACT_WAKE_RESOURCE, now)) status |= TRIAL_ERR_FEL_OVERFLOW;
    }

    // the same three with priorities (PRE): the waiter's entry goes into the guard's heap under a fresh sequence number ...
    CMB_FN void guard_wait_cmd(static_heap_guard<NPROC> &g, uint32_t pid, uint32_t, int32_t)
    {
        const uint32_t s = ++guard_seq;
        at_process(pid, [&](int i) { this->gkey[i] = s; });
        if (!g.push(now, s, prio_of(pid), pid)) status |= TRIAL_ERR_GUARD_OVERFLOW;
        cmd = CMD_NONE;
    }

    // ... a waiter woken by anything but the guard takes its entry out (:153-162) ...
    CMB_FN int64_t guard_wait_end(static_heap_guard<NPROC> &g, uint32_t pid, int64_t sig)
    {
        if (sig != CMB_PROCESS_SUCCESS) {
            uint32_t key = 0u;
            at_process(pid, [&](int i) { key = this->gkey[i]; });
            g.remove(key);
        }
        return sig;
    }

    // ... and a signal wakes whoever is at the top of the heap, at its process's priority now
    CMB_FN void guard_signal(static_heap_guard<NPROC> &g, bool ok)
    {
        if (g.count == 0u || !ok) return;
        const uint32_t head = g.e[1].subj;
        g.pop();
        if (!fel.schedule((int)head, ACT_WAKE_RESOURCE, now, prio_of(head))) status |= TRIAL_ERR_FEL_OVERFLOW;
    }

    // cmb_condition_wait up to its yield (src/cmb_condition.c:63-80): the waiter and its predicate go into the condition's heap,
    // in either form
    CMB_FN void guard_wait_cmd(condition_guard &g, uint32_t pid, uint32_t demand, int32_t ctx)
    {
        const uint32_t s = ++guard_seq;
        if constexpr (PRE) at_process(pid, [&](int i) { this->gkey[i] = s; });
        static_condition_entry x;
        x.d = now;
        x.key = s;
        x.prio = prio_of(pid);
        x.subj = pid;
        x.demand = demand;
        x.ctx = ctx;
        if (!g.push(x)) status |= TRIAL_ERR_GUARD_OVERFLOW;
        cmd = CMD_NONE;
    }

    // ... woken by anything but the signal (only an interrupt can, so only in the second form), the waiter takes its entry out
    CMB_FN int64_t guard_wait_end(condition_guard &g, uint32_t pid, int64_t sig)
    {
        if (sig != CMB_PROCESS_SUCCESS) {
            if constexpr (PRE) {
                uint32_t key = 0u;
                at_process(pid, [&](int i) { key = this->gkey[i]; });
                g.remove(key);
            }
            else {
                status |= TRIAL_ERR_PROC_OVERFLOW;
            }
        }
        return sig;
    }
};

// cmb::Sim::fel_high - the deepest the event list was when an event was taken (cmb_device.cuh's execute) - for a model that says
// `static constexpr bool static_fel_high = true;` (it reports it).  A class of its own around the tier's StaticSim, so that models
// without the trait keep their layout; the free functions below take it as it is, so that a model's demand() gets its own sim.
template <class Base>
struct StaticSimHigh : Base {
    uint32_t fel_high;

    template <class... A>
    CMB_FN void init(A... a)
    {
        Base::init(a...);
        fel_high = 0u;
    }
};

template <class Model, class = void>
struct StaticFelHigh {
    static constexpr bool value = false;
};
template <class Model>
struct StaticFelHigh<Model, typename std::enable_if<Model::static_fel_high>::type> {
    static constexpr bool value = true;
};

// The free functions below take the model's own sim as `class S` - a StaticSim, or the StaticSimHigh around it - and read its
// form from S::PROCESSES, S::INTERRUPTS and S::WAITS.  Those that take nothing else of the tier's would also match cmb::Sim, or
// distributions.cuh's GpDraws, and outrank or shadow the overloads meant for them: they are constrained to the tier's sims.
template <class S>
struct IsStaticSim : std::false_type {
};
template <int NPROC, int NQUEUE, int NEVENT, bool PRE, bool W>
struct IsStaticSim<StaticSim<NPROC, NQUEUE, NEVENT, PRE, W>> : std::true_type {
};
template <class Base>
struct IsStaticSim<StaticSimHigh<Base>> : std::true_type {
};
template <class S>
using if_static_sim = typename std::enable_if<IsStaticSim<S>::value, int>::type;

// cmb_random_exponential / cmb_random_normal in a process body: inline (a call would take the generator's address and put the
// whole control block in local memory)
// In a sampler the dispatcher is trying out (hot_only), a draw that leaves its ziggurat's rectangles gives up - the dispatcher
// rewinds the generator and repeats the whole sampler later, slow paths allowed, together with other lanes in the same position.
template <class S, if_static_sim<S> = 0>
CMB_FN double draw_exponential(S &sim, double mean)                                 // include/cmb_random.h:319-352
{
    if (sim.hot_failed) return mean;
    const uint64_t u = sim.rng.next();
    if (Sfc64::exp_is_hot(u)) return __dmul_rn(mean, Sfc64::exp_hot(*sim.hot, u));
    if (sim.hot_only) {
        sim.hot_failed = true;
        return mean;
    }
    return __dmul_rn(mean, sim.rng.exp_cold(u));
}

template <class S, if_static_sim<S> = 0>
CMB_FN double draw_std_normal(S &sim)                                               // include/cmb_random.h:206-215
{
    if (sim.hot_failed) return 1.0;
    const int64_t ix = (int64_t)sim.rng.next();
    const unsigned i = (unsigned)(ix & 0xff);
    if (i <= ZIG_NOR_MAX) return __dmul_rn(sim.hot->nor_x[i], __ll2double_rn(ix));
    if (sim.hot_only) {
        sim.hot_failed = true;
        return 1.0;
    }
    return sim.rng.nor_cold(*sim.hot, ix);
}

// ------------------------------------------------------------------------------------------------ observers
// cmb_resourceguard_register(g, obs) (cmb_device.cuh's guard_register): with W, a cmb_condition's guard may observe any other
// guard, STATIC_OBSERVERS links in all.  A third observer of one guard replaces its second, as cmb::Sim's does.  Anything else -
// another kind of observer, more links, or no W - sends the trial to the general engine.
template <class Model, class S, class G, class O, if_static_sim<S> = 0>
CMB_FN void guard_register(S &sim, Model &, G &, O &)
{
    sim.status |= TRIAL_ERR_PROC_OVERFLOW;
}

template <class Model, class S, class G, if_static_sim<S> = 0>
CMB_FN void guard_register(S &sim, Model &, G &g, static_heap_guard<S::PROCESSES, static_condition_entry> &obs)
{
    if constexpr (S::WAITS) {
        uint32_t mine = 0u, last = 0u;
        for (uint32_t k = 0u; k < sim.nobs; k++) {
            if (sim.obs_from[k] == (const void *)&g) {
                mine++;
                last = k;
            }
        }
        if (mine >= 2u) {
            sim.obs_to[last] = &obs;
        }
        else if (sim.nobs < (uint32_t)STATIC_OBSERVERS) {
            sim.obs_from[sim.nobs] = (const void *)&g;
            sim.obs_to[sim.nobs] = &obs;
            sim.nobs++;
        }
        else {
            sim.status |= TRIAL_ERR_PROC_OVERFLOW;
        }
    }
    else {
        (void)g;
        (void)obs;
        sim.status |= TRIAL_ERR_PROC_OVERFLOW;
    }
}

// cmb_resourceguard_signal (src/cmb_resourceguard.c:202-242, cmb_device.cuh's guard_signal): the guard's own head first, then
// each observer's head only, if its predicate holds - even when the guard had nobody to wake.  An observer's wake-up takes the
// waiter's own event slot, as cmb_condition_signal's does.  An observer that is itself observed would need the general engine's
// recursion: the trial goes there.
template <class Model, class S, class G>
CMB_FN void static_guard_signal(S &sim, Model &m, G &g, bool ok)
{
    sim.guard_signal(g, ok);
    if constexpr (S::WAITS) {
        for (uint32_t k = 0u; k < sim.nobs; k++) {
            if (sim.obs_from[k] != (const void *)&g) continue;
            auto &o = *sim.obs_to[k];
            for (uint32_t j = 0u; j < sim.nobs; j++) {
                if (sim.obs_from[j] == (const void *)&o) sim.status |= TRIAL_ERR_PROC_OVERFLOW;
            }
            if (o.count == 0u) continue;
            const static_condition_entry head = o.e[1];
            if (m.demand(sim, head.demand, head.subj, head.ctx)) {
                o.pop();
                if (!sim.fel.schedule((int)head.subj, ACT_WAKE_RESOURCE, sim.now, sim.prio_of(head.subj))) sim.status |= TRIAL_ERR_FEL_OVERFLOW;
            }
        }
    }
    else {
        (void)m;
    }
}

// ------------------------------------------------------------------------------------------------ objectqueue
template <class S, bool RECORD>
CMB_FN void objectqueue_initialize(S &sim, static_objectqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t capacity)
{
    uint32_t k = sim.nqueue;
    if (k >= (uint32_t)S::QUEUES) {
        sim.status |= TRIAL_ERR_PROC_OVERFLOW;
        k = 0u;
    }
    sim.nqueue = k + 1u;
    q.rear.reset();
    q.front.reset();
    q.ring.init(sim.ring_win + (size_t)k * STATIC_WINDOW * sim.ring_stride, sim.ring_stride,
                sim.spill_cap ? sim.spill + (size_t)k * sim.spill_cap : nullptr, sim.spill_cap);
    q.capacity = capacity;
    q.longest = 0u;
    q.length = 0u;
    if constexpr (RECORD) q.recording = 0u;
}

template <class S>
CMB_FN void objectqueue_recording_start(S &sim, static_objectqueue<S::PROCESSES, true, S::INTERRUPTS> &q) { q.start(sim); }
template <class S>
CMB_FN void objectqueue_recording_stop(S &sim, static_objectqueue<S::PROCESSES, true, S::INTERRUPTS> &q) { q.stop(sim); }

template <class Model, class S, bool RECORD>
CMB_FN bool objectqueue_try_put(S &sim, Model &m, static_objectqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t obj)
{
    if ((uint64_t)q.ring.len >= q.capacity) return false;
    if (!q.ring.put(__longlong_as_double((long long)obj))) sim.status |= TRIAL_ERR_QUEUE_OVERFLOW;     // void from here on: re-run
    q.longest = q.ring.len > q.longest ? q.ring.len : q.longest;
    q.length = q.ring.len;
    q.sample(sim);                                      // record_sample in put, :289
    static_guard_signal(sim, m, q.front, true);
    return true;
}

template <class Model, class S, bool RECORD>
CMB_FN bool objectqueue_try_get(S &sim, Model &m, static_objectqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t &obj)
{
    if (q.ring.len == 0u) return false;
    obj = (uint64_t)__double_as_longlong(q.ring.take());
    q.length = q.ring.len;
    q.sample(sim);                                      // ... and in get, :226-229
    static_guard_signal(sim, m, q.rear, true);
    return true;
}

// ------------------------------------------------------------------------------------------------ buffer
template <class S, bool RECORD>
CMB_FN void buffer_initialize(S &, static_buffer<S::PROCESSES, RECORD, S::INTERRUPTS> &b, uint64_t capacity)
{
    b.rear.reset();
    b.front.reset();
    b.level = 0u;
    b.capacity = capacity;
    if constexpr (RECORD) b.recording = 0u;
}

template <class S>
CMB_FN void buffer_recording_start(S &sim, static_buffer<S::PROCESSES, true, S::INTERRUPTS> &b) { b.start(sim); }
template <class S>
CMB_FN void buffer_recording_stop(S &sim, static_buffer<S::PROCESSES, true, S::INTERRUPTS> &b) { b.stop(sim); }

// cmb_buffer_get / cmb_buffer_put up to their waits, as cmb_device.cuh's buffer_get_step / buffer_put_step (src/cmb_buffer.c:194-346)
template <class Model, class S, bool RECORD>
CMB_FN bool buffer_get_step(S &sim, Model &m, static_buffer<S::PROCESSES, RECORD, S::INTERRUPTS> &b, uint32_t pid)
{
    uint64_t rem = 0u, got = 0u;
    sim.at_process(pid, [&](int i) {
        rem = sim.proc[i].fr[1];
        got = sim.proc[i].fr[2];
    });
    bool done;
    if (b.level >= rem) {
        b.level -= rem;
        b.sample(sim);
        got += rem;
        static_guard_signal(sim, m, b.rear, b.level < b.capacity);
        if (b.level > 0u) static_guard_signal(sim, m, b.front, true);
        done = true;
    }
    else {
        if (b.level > 0u) {
            const uint64_t grab = b.level;
            b.level = 0u;
            b.sample(sim);
            got += grab;
            rem -= grab;
            static_guard_signal(sim, m, b.rear, b.level < b.capacity);
        }
        static_guard_signal(sim, m, b.rear, b.level < b.capacity);
        done = false;
    }
    sim.at_process(pid, [&](int i) {
        sim.proc[i].fr[1] = rem;
        sim.proc[i].fr[2] = got;
    });
    return done;
}

template <class Model, class S, bool RECORD>
CMB_FN bool buffer_put_step(S &sim, Model &m, static_buffer<S::PROCESSES, RECORD, S::INTERRUPTS> &b, uint32_t pid)
{
    uint64_t rem = 0u;
    sim.at_process(pid, [&](int i) { rem = sim.proc[i].fr[1]; });
    bool done;
    if (b.capacity - b.level >= rem) {
        b.level += rem;
        b.sample(sim);
        rem = 0u;
        static_guard_signal(sim, m, b.front, b.level > 0u);
        if (b.level < b.capacity) static_guard_signal(sim, m, b.rear, true);
        done = true;
    }
    else {
        if (b.level < b.capacity) {
            const uint64_t grab = b.capacity - b.level;
            b.level = b.capacity;
            b.sample(sim);
            rem -= grab;
            static_guard_signal(sim, m, b.front, b.level > 0u);
        }
        static_guard_signal(sim, m, b.front, b.level > 0u);
        done = false;
    }
    sim.at_process(pid, [&](int i) { sim.proc[i].fr[1] = rem; });
    return done;
}

// ------------------------------------------------------------------------------------------------ resourcepool
// as cmb_device.cuh's functions of the same names (src/cmb_resourcepool.c), the holders' records in registers.  Every waiter
// wants units (DEMAND_POOL_AVAILABLE), so a signal's demand is `capacity - in_use > 0`.
template <class S, bool RECORD>
CMB_FN void resourcepool_initialize(S &, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint64_t capacity)
{
    rp.guard.reset();
#pragma unroll
    for (int i = 0; i < S::PROCESSES; i++) rp.held[i] = 0u;
    rp.capacity = capacity;
    rp.in_use = 0u;
    rp.holding = 0u;
    if constexpr (RECORD) rp.recording = 0u;
}

template <class S>
CMB_FN void resourcepool_recording_start(S &sim, static_resourcepool<S::PROCESSES, true, S::INTERRUPTS> &rp) { rp.start(sim); }
template <class S>
CMB_FN void resourcepool_recording_stop(S &sim, static_resourcepool<S::PROCESSES, true, S::INTERRUPTS> &rp) { rp.stop(sim); }

template <class S, bool RECORD>
CMB_FN uint64_t resourcepool_held_by_process(S &sim, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint32_t pid)
{
    uint64_t h = 0u;
    sim.at_process(pid, [&](int i) { h = rp.held[i]; });
    return h;
}

// update_record (src/cmb_resourcepool.c:324-355): the caller's record grows by `amount`, made if it had none
template <class S, bool RECORD>
CMB_FN void pool_update_record(S &sim, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint32_t pid, uint64_t amount)
{
    sim.at_process(pid, [&](int i) {
        if (((rp.holding >> i) & 1u) == 0u) {
            rp.holding |= 1u << i;
            sim.holds_add(pid, 1);
        }
        rp.held[i] += amount;
    });
}

// pid's holder record leaves the pool (its units stay counted in in_use); returns the amount it held
template <class S, bool RECORD>
CMB_FN uint64_t pool_take_record(S &sim, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint32_t pid)
{
    uint64_t h = 0u;
    sim.at_process(pid, [&](int i) {
        if (((rp.holding >> i) & 1u) != 0u) {
            h = rp.held[i];
            rp.held[i] = 0u;
            rp.holding &= ~(1u << i);
            sim.holds_add(pid, -1);
        }
    });
    return h;
}

// cmi_pool_acquire_inner up to its wait (:362-497): true = satisfied, false = the caller waits at the guard for the rest.
// fr[1] = the remaining claim.  A grab that leaves the claim unmet keeps what it took (the greedy partial grab).
// cmb_resourcepool_preempt then takes from holders of lower priority, the lowest first (:425-476), which needs PRE; without
// it the trial goes to the general engine.
template <class Model, class S, bool RECORD>
CMB_FN bool pool_acquire_step(S &sim, Model &m, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint32_t pid, bool preempt)
{
    if constexpr (!S::INTERRUPTS) {
        if (preempt) sim.status |= TRIAL_ERR_PROC_OVERFLOW;
    }
    uint64_t rem = 0u;
    sim.at_process(pid, [&](int i) { rem = sim.proc[i].fr[1]; });
    const uint64_t available = rp.capacity - rp.in_use;
    if (available >= rem) {
        rp.in_use += rem;
        rp.sample(sim);
        pool_update_record(sim, rp, pid, rem);
        static_guard_signal(sim, m, rp.guard, rp.capacity - rp.in_use > 0u);
        return true;
    }
    if (available > 0u) {
        rp.in_use += available;
        rp.sample(sim);
        rem -= available;
        pool_update_record(sim, rp, pid, available);
    }
    if constexpr (S::INTERRUPTS) {
        const int32_t mine = sim.prio_of(pid);
        while (preempt) {
            // the top of the holders' heap under HolderOrder - lowest priority, then the larger key (process index + 1,
            // SURVEY.md quirk 4) - a strict order, so the selection over the holder bits is the heap's top exactly
            int victim = -1;
            int32_t vp = 0;
#pragma unroll
            for (int i = 0; i < S::PROCESSES; i++) {
                const int32_t p = sim.prio_of((uint32_t)i);
                if (((rp.holding >> i) & 1u) != 0u && (victim < 0 || p <= vp)) {
                    victim = i;
                    vp = p;
                }
            }
            if (victim < 0 || vp >= mine) break;
            const uint64_t loot = pool_take_record(sim, rp, (uint32_t)victim);
            sim.interrupt((uint32_t)victim, CMB_PROCESS_PREEMPTED, vp);
            if (loot < rem) {
                pool_update_record(sim, rp, pid, loot);
                rem -= loot;
            }
            else {
                pool_update_record(sim, rp, pid, rem);
                rp.in_use -= loot - rem;
                rp.sample(sim);
                static_guard_signal(sim, m, rp.guard, rp.capacity - rp.in_use > 0u);
                rem = 0u;
                break;
            }
        }
    }
    sim.at_process(pid, [&](int i) { sim.proc[i].fr[1] = rem; });
    if constexpr (S::INTERRUPTS) return rem == 0u;
    return false;
}

// the tail of cmi_pool_acquire_inner after an unsuccessful wait (:499-531): back to the holding at the call.  Only an
// interrupt, a timer or a pre-emption ends a wait unsuccessfully; without PRE none of them exists on this tier, and should one
// ever get here, the general engine answers.
template <class Model, class S, bool RECORD>
CMB_FN void pool_acquire_rollback(S &sim, Model &m, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint32_t pid, int64_t sig)
{
    if constexpr (S::INTERRUPTS) {
        if (sig == CMB_PROCESS_PREEMPTED) return;       // thrown out: returns empty-handed, nothing to unwind
        uint64_t initially = 0u;
        sim.at_process(pid, [&](int i) { initially = sim.proc[i].fr[0]; });
        if (initially > 0u) {                           // reset_holder
            uint64_t surplus = 0u;
            sim.at_process(pid, [&](int i) {
                if (((rp.holding >> i) & 1u) != 0u) {
                    surplus = rp.held[i] - initially;
                    rp.held[i] = initially;
                }
            });
            rp.in_use -= surplus;
            rp.sample(sim);
            static_guard_signal(sim, m, rp.guard, rp.capacity - rp.in_use > 0u);
        }
        else {
            rp.in_use -= resourcepool_held_by_process(sim, rp, pid);
            rp.sample(sim);
            (void)pool_take_record(sim, rp, pid);
        }
    }
    else {
        sim.status |= TRIAL_ERR_PROC_OVERFLOW;
    }
}

// cmb_resourcepool_release, :561-605
template <class Model, class S, bool RECORD>
CMB_FN void resourcepool_release(S &sim, Model &m, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint32_t pid, uint64_t amount)
{
    sim.at_process(pid, [&](int i) {
        if (((rp.holding >> i) & 1u) != 0u) {
            if (rp.held[i] == amount) {
                rp.holding &= ~(1u << i);
                sim.holds_add(pid, -1);
                rp.held[i] = 0u;
            }
            else {
                rp.held[i] -= amount;
            }
        }
    });
    rp.in_use -= amount;
    rp.sample(sim);
    static_guard_signal(sim, m, rp.guard, rp.capacity - rp.in_use > 0u);
}

// ------------------------------------------------------------------------------------------------ resource
// as cmb_device.cuh's (src/cmb_resource.c); every waiter wants it free (DEMAND_RESOURCE_FREE)
template <class S, bool RECORD>
CMB_FN void resource_initialize(S &, static_resource<S::PROCESSES, RECORD, S::INTERRUPTS> &r)
{
    r.guard.reset();
    r.holder = NIL;
    if constexpr (RECORD) r.recording = 0u;
}

// record_sample; CMB_RESOURCE_ACQUIRE calls it too
template <class S, bool RECORD>
CMB_FN void resource_sample(S &sim, static_resource<S::PROCESSES, RECORD, S::INTERRUPTS> &r) { r.sample(sim); }

template <class S>
CMB_FN void resource_recording_start(S &sim, static_resource<S::PROCESSES, true, S::INTERRUPTS> &r) { r.start(sim); }
template <class S>
CMB_FN void resource_recording_stop(S &sim, static_resource<S::PROCESSES, true, S::INTERRUPTS> &r) { r.stop(sim); }

template <class S, bool RECORD>
CMB_FN void resource_grab(S &sim, static_resource<S::PROCESSES, RECORD, S::INTERRUPTS> &r, uint32_t pid)     // :182-189
{
    r.holder = pid;
    sim.holds_add(pid, 1);
}

template <class Model, class S, bool RECORD>
CMB_FN void resource_release(S &sim, Model &m, static_resource<S::PROCESSES, RECORD, S::INTERRUPTS> &r, uint32_t pid)  // :234-250
{
    if (r.holder == pid) sim.holds_add(pid, -1);
    r.holder = NIL;
    resource_sample(sim, r);
    static_guard_signal(sim, m, r.guard, true);
}

// cmb_resource_preempt, :270-320, up to its polite branch, as cmb_device.cuh's resource_preempt_step: a holder of equal or
// lower priority is evicted by an ACT_CMB_WAKE_PREEMPT (a spare slot) and the CALLER's awaiteds are cancelled (sic).  true =
// the caller holds the resource now; false = go on as cmb_resource_acquire.  Without PRE the trial goes to the general engine
// (and is void by then, but runs to its end like any flagged trial).
template <class S, bool RECORD>
CMB_FN bool resource_preempt_step(S &sim, static_resource<S::PROCESSES, RECORD, S::INTERRUPTS> &r, uint32_t pid)
{
    if constexpr (S::INTERRUPTS) {
        const uint32_t victim = r.holder;
        if (victim == NIL) {
            resource_grab(sim, r, pid);
            resource_sample(sim, r);
            return true;
        }
        if (sim.prio_of(pid) >= sim.prio_of(victim)) {
            sim.holds_add(victim, -1);
            sim.cancel_awaiteds(pid);
            r.holder = NIL;
            (void)sim.schedule(ACT_CMB_WAKE_PREEMPT, victim, CMB_PROCESS_PREEMPTED, sim.now, sim.prio_of(victim));
            resource_grab(sim, r, pid);                 // no history sample: the resource stays occupied
            return true;
        }
        return false;
    }
    else {
        (void)r;
        (void)pid;
        sim.status |= TRIAL_ERR_PROC_OVERFLOW;
        return false;
    }
}

// cmb_process_priority_set (src/cmb_process.c:150-198, as cmb_device.cuh's): the process's pending wake-up from a hold moves in
// the event list; its holder records follow by themselves (they carry its priority); a guard entry keeps the old one (SURVEY.md
// quirk 2).  Without PRE a priority other than 0 goes to the general engine.
template <class S, if_static_sim<S> = 0>
CMB_FN void process_priority_set(S &sim, uint32_t pid, int64_t pri)
{
    if constexpr (S::INTERRUPTS) {
        sim.at_process(pid, [&](int i) {
            sim.prio[i] = (int32_t)pri;
            if ((sim.fel.key[i] & 3u) == ACT_WAKE_TIME) sim.fel.prio[i] = (int32_t)pri;
        });
    }
    else if (pri != 0) {
        sim.status |= TRIAL_ERR_PROC_OVERFLOW;
    }
}

// cmb_process_priority (0 in the tier's first form)
template <class S, if_static_sim<S> = 0>
CMB_FN int64_t process_priority(const S &sim, uint32_t pid)
{
    return (int64_t)sim.prio_of(pid);
}

// ------------------------------------------------------------------------------------------------ priorityqueue
// as cmb_device.cuh's functions of the same names (src/cmb_priorityqueue.c), over the table
template <class S, bool RECORD>
CMB_FN void priorityqueue_initialize(S &, static_priorityqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t capacity)
{
    q.rear.reset();
    q.front.reset();
    q.capacity = capacity;
    q.issued = 0u;
    q.count = 0u;
    if constexpr (RECORD) q.recording = 0u;
}

template <int NPROC, bool RECORD, bool PRE>
CMB_FN uint64_t priorityqueue_length(const static_priorityqueue<NPROC, RECORD, PRE> &q)
{
    return (uint64_t)q.count;
}

template <class S>
CMB_FN void priorityqueue_recording_start(S &sim, static_priorityqueue<S::PROCESSES, true, S::INTERRUPTS> &q) { q.start(sim); }
template <class S>
CMB_FN void priorityqueue_recording_stop(S &sim, static_priorityqueue<S::PROCESSES, true, S::INTERRUPTS> &q) { q.stop(sim); }

// PrioOrder (src/cmb_priorityqueue.c:43-54): a strict total order, handles being unique
CMB_FN bool static_pq_before(const static_pq_entry &a, const static_pq_entry &b)
{
    if (a.prio != b.prio) return a.prio > b.prio;
    return a.handle < b.handle;
}

// the table index of `handle`, -1 if it is not in the queue
template <int NPROC, bool RECORD, bool PRE>
CMB_FN int static_pq_find(const static_priorityqueue<NPROC, RECORD, PRE> &q, uint64_t handle)
{
    int at = -1;
    for (uint32_t k = 0u; k < q.count; k++) {
        if (q.e[k].handle == handle) at = (int)k;
    }
    return at;
}

// the entry at `at` leaves; the last one takes its place (the table is unsorted)
template <int NPROC, bool RECORD, bool PRE>
CMB_FN void static_pq_take(static_priorityqueue<NPROC, RECORD, PRE> &q, int at)
{
    q.count--;
    q.e[at] = q.e[q.count];
}

template <class Model, class S, bool RECORD>
CMB_FN bool priorityqueue_try_put(S &sim, Model &m, static_priorityqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t obj, int64_t prio,
                                  uint64_t *handle)                                 // :237-284
{
    if ((uint64_t)q.count >= q.capacity) return false;
    const uint64_t h = ++q.issued;
    if (q.count >= (uint32_t)STATIC_PQ_CAP) {
        sim.status |= TRIAL_ERR_QUEUE_OVERFLOW;         // void from here on: re-run
    }
    else {
        q.e[q.count].obj = obj;
        q.e[q.count].handle = h;
        q.e[q.count].prio = (int32_t)prio;
        q.count++;
    }
    if (handle != nullptr) *handle = h;
    q.sample(sim);
    static_guard_signal(sim, m, q.front, true);
    return true;
}

template <class Model, class S, bool RECORD>
CMB_FN bool priorityqueue_try_get(S &sim, Model &m, static_priorityqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t &obj)   // :189-235
{
    if (q.count == 0u) return false;
    int best = 0;
    for (uint32_t k = 1u; k < q.count; k++) {
        if (static_pq_before(q.e[k], q.e[best])) best = (int)k;
    }
    obj = q.e[best].obj;
    static_pq_take(q, best);
    q.sample(sim);
    static_guard_signal(sim, m, q.rear, true);
    return true;
}

// cmb_priorityqueue_position, :286-320: 1 = next to be taken, 0 = not in the queue
template <class S, bool RECORD>
CMB_FN uint64_t priorityqueue_position(S &, static_priorityqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t handle)
{
    const int at = static_pq_find(q, handle);
    if (at < 0) return 0u;
    uint64_t ahead = 0u;
    for (uint32_t k = 0u; k < q.count; k++) {
        if (static_pq_before(q.e[k], q.e[at])) ahead++;
    }
    return ahead + 1u;
}

// cmb_priorityqueue_cancel: the object leaves without a signal or a history sample, as on the general engine
template <class S, bool RECORD>
CMB_FN bool priorityqueue_cancel(S &, static_priorityqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t handle)
{
    const int at = static_pq_find(q, handle);
    if (at < 0) return false;
    static_pq_take(q, at);
    return true;
}

// cmb_priorityqueue_reprioritize, include/cmb_priorityqueue.h:170-180: the object and its handle stay
template <class S, bool RECORD>
CMB_FN void priorityqueue_reprioritize(S &, static_priorityqueue<S::PROCESSES, RECORD, S::INTERRUPTS> &q, uint64_t handle, int64_t prio)
{
    const int at = static_pq_find(q, handle);
    if (at >= 0) q.e[at].prio = (int32_t)prio;
}

// ------------------------------------------------------------------------------------------------ condition
template <class S>
CMB_FN void condition_initialize(S &, static_condition<S::PROCESSES> &c)
{
    c.guard.reset();
}

// cmb_condition_signal, src/cmb_condition.c:120-167, as cmb_device.cuh's: every waiter whose predicate holds, in heap-array
// order, is woken at `now` with its process's priority; the hits leave the heap in a second pass, in the order they were found.
// The wake-up goes into the waiter's own event slot - empty while it waits - as ACT_WAKE_RESOURCE, which resumes a running
// process with CMB_PROCESS_SUCCESS exactly as ACT_CMB_WAKE_CONDITION does: no spare slot is needed, and an interrupt that pops
// first drops it with the rest of the process's slot (cancel_awaiteds), as the general engine's pattern cancel does.
template <class Model, class S>
CMB_FN uint32_t condition_signal(S &sim, Model &m, static_condition<S::PROCESSES> &c)
{
    auto &h = c.guard;
    if (h.count == 0u) return 0u;
    uint32_t hit[S::PROCESSES];
    uint32_t n = 0u;
    for (uint32_t k = 1u; k <= h.count; k++) {
        const uint32_t pid = h.e[k].subj;
        if (m.demand(sim, h.e[k].demand, pid, h.e[k].ctx)) {
            hit[n++] = h.e[k].key;
            if (!sim.fel.schedule((int)pid, ACT_WAKE_RESOURCE, sim.now, sim.prio_of(pid))) sim.status |= TRIAL_ERR_FEL_OVERFLOW;
        }
    }
    for (uint32_t k = 0u; k < n; k++) h.remove(hit[k]);
    return n;
}

// ------------------------------------------------------------------------------------------------ process end
// A model of the tier's second form may name the pools and resources its processes can hold from:
//   template <class F> CMB_FN void static_holdables(F &&visit) { visit(cheese); }
// The tier then drops the holdings of a process that is stopped or exits, as cmi_process_drop_resources does (src/cmb_process.c:
// 507-527).  One holding at most: the reference drops several in the reverse order of their acquisition, which the tier does not
// keep, so a process that ends holding from two or more containers sends the trial to the general engine.
struct StaticHoldablesProbe {
    template <class C>
    CMB_FN void operator()(C &) const {}
};
template <class Model, class = void>
struct StaticHoldables {
    static constexpr bool known = false;
};
template <class Model>
struct StaticHoldables<Model, decltype(std::declval<Model &>().static_holdables(StaticHoldablesProbe{}))> {
    static constexpr bool known = true;
};

// pool_drop_holder (src/cmb_resourcepool.c:98-121): no history sample, as there
template <class Model, class S, bool RECORD>
CMB_FN void static_drop_holder(S &sim, Model &m, static_resourcepool<S::PROCESSES, RECORD, S::INTERRUPTS> &rp, uint32_t pid)
{
    if (((rp.holding >> pid) & 1u) == 0u) return;
    rp.in_use -= pool_take_record(sim, rp, pid);
    static_guard_signal(sim, m, rp.guard, rp.capacity - rp.in_use > 0u);
}

// resource_drop_holder (src/cmb_resource.c:45-56)
template <class Model, class S, bool RECORD>
CMB_FN void static_drop_holder(S &sim, Model &m, static_resource<S::PROCESSES, RECORD, S::INTERRUPTS> &r, uint32_t pid)
{
    if (r.holder != pid) return;
    sim.holds_add(pid, -1);
    r.holder = NIL;
    resource_sample(sim, r);
    static_guard_signal(sim, m, r.guard, true);
}

template <class Model, class S>
CMB_FN void static_drop_resources(S &sim, Model &m, uint32_t pid)
{
    if constexpr (S::INTERRUPTS && StaticHoldables<Model>::known) {
        const uint32_t n = sim.holds_of(pid);
        if (n > 1u) sim.status |= TRIAL_ERR_PROC_OVERFLOW;
        else if (n == 1u) m.static_holdables([&](auto &c) { static_drop_holder(sim, m, c, pid); });
    }
}

// cmb_process_stop (src/cmb_process.c:698-723) as far as this tier can need it: the process's pending event goes, it is
// FINISHED; an entry it may have in a guard stays (SURVEY.md quirk 2) and will swallow one signal.  PRE: its interrupts and
// pre-emptions go too, and its holdings are dropped (static_drop_resources).  Otherwise a process stopped while it holds from
// a pool or a resource would drop its holdings: static_trial_end flags that.
template <class Model, class S, if_static_sim<S> = 0>
CMB_FN void process_stop(S &sim, Model &m, uint32_t pid, int64_t value)
{
    if constexpr (S::INTERRUPTS) {
        bool running = false;
        sim.at_process(pid, [&](int i) {
            if (sim.proc[i].status == PROC_RUNNING) {
                running = true;
                sim.proc[i].status = PROC_FINISHED;
                sim.proc[i].exit_value = value;
            }
        });
        if (!running) return;
        sim.cancel_awaiteds(pid);
        static_drop_resources(sim, m, pid);
        if constexpr (S::WAITS) sim.wake_process_waiters(pid, CMB_PROCESS_STOPPED);
        return;
    }
    (void)m;
    sim.at_process(pid, [&](int i) {
        if (sim.proc[i].status == PROC_RUNNING) {
            sim.proc[i].status = PROC_FINISHED;
            sim.proc[i].exit_value = value;
            sim.fel.drop(i);
        }
    });
}

// ------------------------------------------------------------------------------------------------ dispatcher
// A model may state the kinds of its processes in creation order - `static CMB_FN constexpr uint32_t static_kind(uint32_t i)` -
// and the dispatcher then knows at compile time which body process i runs (one copy of each body instead of NPROC, no run-time
// branch on the kind); a trial whose cmb_process_create calls disagree with the table is flagged and goes to the general engine.
template <class Model, class = void>
struct StaticKinds {
    static constexpr bool known = false;
    template <int I>
    static CMB_FN uint32_t of(uint32_t runtime_kind) { return runtime_kind; }
    template <class S>
    static CMB_FN bool agree(const S &) { return true; }
};
template <class Model>
struct StaticKinds<Model, decltype((void)Model::static_kind(0u))> {
    static constexpr bool known = true;
    template <int I>
    static CMB_FN uint32_t of(uint32_t) { return Model::static_kind((uint32_t)I); }
    template <class S>
    static CMB_FN bool agree(const S &sim)
    {
        return agree_from<S, 0>(sim);
    }
    template <class S, int I>
    static CMB_FN bool agree_from(const S &sim)
    {
        if constexpr (I < S::PROCESSES) {
            return ((uint32_t)I >= sim.nproc || sim.proc[I].kind == Model::static_kind((uint32_t)I)) && agree_from<S, I + 1>(sim);
        }
        else {
            return true;
        }
    }
};

// S: the StaticSim the model was instantiated over (StaticSimHigh<StaticSim<...>> for a model with static_fel_high)
template <class Model, class S, int I, int NPROC = S::PROCESSES>
struct StaticDispatch {
    static CMB_FN void run(S &sim, Model &m, int who, int64_t sig)
    {
        if (who == I) m.process(sim, (uint32_t)I, StaticKinds<Model>::template of<I>(sim.proc[I].kind), sig);
        else StaticDispatch<Model, S, I + 1>::run(sim, m, who, sig);
    }
};
template <class Model, class S, int NPROC>
struct StaticDispatch<Model, S, NPROC, NPROC> {
    static CMB_FN void run(S &, Model &, int, int64_t) {}
};

// one step of cmb_event_queue_execute (src/cmb_event.c:229-252): pop, advance the clock, resume the process.  false = the
// list ran dry.  The body's blocking call is left in sim.cmd for the caller (`who` = the process it belongs to).
template <class Model, class S>
CMB_FN bool static_step(S &sim, Model &m, int &who)
{
    constexpr int NPROC = S::PROCESSES, NEVENT = S::SLOTS - S::PROCESSES;
    constexpr bool PRE = S::INTERRUPTS;
    uint32_t act, key;
    double when;
    if constexpr (StaticFelHigh<Model>::value) {
        uint32_t depth = 0u;
#pragma unroll
        for (int i = 0; i < S::SLOTS; i++) depth += sim.fel.key[i] != 0u ? 1u : 0u;
        if (depth > sim.fel_high) sim.fel_high = depth;
    }
    if (!sim.fel.pop(who, act, when, key)) return false;
    sim.now = when;
    sim.current_event = key;
    sim.pops++;
    sim.cmd = CMD_NONE;
    if constexpr (PRE) {
        if (who >= NPROC) {
            uint32_t uact = 0u, subj = 0u;
            int64_t arg = 0;
#pragma unroll
            for (int i = 0; i < NEVENT; i++) {
                if (i == who - NPROC) {
                    uact = sim.uev[i].act;
                    subj = sim.uev[i].subj;
                    arg = sim.uev[i].arg;
                }
            }
            if constexpr (S::WAITS) sim.wake_event_waiters(key, CMB_PROCESS_SUCCESS);      // waiters first, src/cmb_event.c:243-249
            if (uact >= ACT_CMB_USER) {
                m.event(sim, uact, subj, arg);
                return true;
            }
            // a process's interrupt (its awaiteds cancelled, the body resumed whatever its state - execute's
            // ACT_CMB_WAKE_INTERRUPT) or a resource pre-emption (resumed if running); the command it ends on is the process's.
            // W: a timer or a resume resumes it whatever its state too; a wake-up from a wait on a process or an event, if running.
            bool run = true;
            if (uact == ACT_CMB_WAKE_INTERRUPT) {
                sim.cancel_awaiteds(subj);
            }
            else if (!(S::WAITS && (uact == ACT_CMB_WAKE_TIME || uact == ACT_CMB_RESUME))) {
                sim.at_process(subj, [&](int i) { run = sim.proc[i].status == PROC_RUNNING; });
            }
            who = (int)subj;
            if (run) {
                sim.current = subj;
                StaticDispatch<Model, S, 0>::run(sim, m, who, arg);
                sim.current = NIL;
            }
            return true;
        }
    }
    if (NEVENT > 0 && who >= NPROC) {                   // an event of the model's own: its action function, no process resumed
#pragma unroll
        for (int i = 0; i < NEVENT; i++) {
            if (i == who - NPROC) m.event(sim, sim.uev[i].act, sim.uev[i].subj, sim.uev[i].arg);
        }
        return true;
    }
    bool run = true;
    sim.at_process((uint32_t)who, [&](int i) {
        if (act == ACT_START) {
            sim.proc[i].status = PROC_RUNNING;
            sim.proc[i].pc = 0u;
        }
        run = sim.proc[i].status == PROC_RUNNING;
    });
    if (run) {
        sim.current = (uint32_t)who;
        StaticDispatch<Model, S, 0>::run(sim, m, who, CMB_PROCESS_SUCCESS);
        sim.current = NIL;
    }
    return true;
}

// The reference drops the holdings of a process that exits or is stopped (cmi_process_drop_resources, src/cmb_process.c:
// 507-527: units back to the pool, the resource freed, their guards signalled); this tier does not.  Only a process itself
// gives back what it holds, so one that ended holding still does when the trial ends - or when it is started again
// (process_start).  Either way the trial goes to the general engine.  Checked here, once per trial, rather than at every exit:
// a model that holds nothing keeps its code.
template <class S>
CMB_FN void static_trial_end(S &sim)
{
    if (sim.holds == 0u) return;
#pragma unroll
    for (int i = 0; i < S::PROCESSES; i++) {
        if (sim.proc[i].status == PROC_FINISHED && sim.holds_of((uint32_t)i) != 0u) sim.status |= TRIAL_ERR_PROC_OVERFLOW;
    }
}

// the blocking call the body ended on, except the holds whose duration the caller draws (exponential, sampled)
template <class Model, class S>
CMB_FN void static_finish_command(S &sim, Model &m, int who, uint32_t cmd)
{
    if (cmd == CMD_HOLD) {
        if (sim.cmd_value < 0.0) sim.status |= TRIAL_ERR_NEGATIVE_HOLD;
        if (!sim.fel.schedule(who, ACT_WAKE_TIME, __dadd_rn(sim.now, sim.cmd_value), sim.prio_of((uint32_t)who)))
            sim.status |= TRIAL_ERR_FEL_OVERFLOW;
    }
    else if (cmd == CMD_EXIT) {                         // cmb_process_exit (:671-684); without W nobody waits for a process
        if constexpr (S::INTERRUPTS) {
            static_drop_resources(sim, m, (uint32_t)who);
            sim.cancel_awaiteds((uint32_t)who);
        }
        if constexpr (S::WAITS) sim.wake_process_waiters((uint32_t)who, CMB_PROCESS_SUCCESS);
        (void)m;
        sim.at_process((uint32_t)who, [&](int i) {
            sim.proc[i].status = PROC_FINISHED;
            sim.proc[i].exit_value = sim.cmd_exit;
        });
    }
}

// cmb_random_flip's cache, where the sim keeps one (StaticSim<..., PRE = true>): the dispatcher saves it with the generator before
// it tries a sampler with the rectangles only, and puts both back when the sampler gives up, so that the repeat sees the flips the
// first try saw
template <class S, class = void>
struct FlipState {
    CMB_FN explicit FlipState(const S &) {}
    CMB_FN void restore(S &) const {}
};
template <class S>
struct FlipState<S, decltype((void)std::declval<S &>().flips)> {
    FlipCache saved;
    CMB_FN explicit FlipState(const S &sim) : saved(sim.flips) {}
    CMB_FN void restore(S &sim) const { sim.flips = saved; }
};

// `static constexpr bool static_interrupts = true;` in a model: its static-tier form is StaticSim<..., PRE = true>
template <class Model, class = void>
struct StaticInterrupts {
    static constexpr bool value = false;
};
template <class Model>
struct StaticInterrupts<Model, typename std::enable_if<Model::static_interrupts>::type> {
    static constexpr bool value = true;
};
// ... and with `static constexpr bool static_waits = true;` as well, StaticSim<..., PRE = true, W = true>
template <class Model, class = void>
struct StaticWaitsOf {
    static constexpr bool value = false;
};
template <class Model>
struct StaticWaitsOf<Model, typename std::enable_if<Model::static_waits>::type> {
    static constexpr bool value = true;
};
template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT>
using StaticFormOf = StaticSim<NPROC, NQUEUE, NEVENT, StaticInterrupts<ModelT<StaticSim<NPROC, NQUEUE, NEVENT>>>::value,
                               StaticInterrupts<ModelT<StaticSim<NPROC, NQUEUE, NEVENT>>>::value
                                   && StaticWaitsOf<ModelT<StaticSim<NPROC, NQUEUE, NEVENT>>>::value>;
// ... and with `static constexpr bool static_fel_high = true;` it also keeps fel_high (StaticSimHigh)
template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT>
using StaticSimOf = typename std::conditional<StaticFelHigh<ModelT<StaticSim<NPROC, NQUEUE, NEVENT>>>::value,
                                              StaticSimHigh<StaticFormOf<ModelT, NPROC, NQUEUE, NEVENT>>,
                                              StaticFormOf<ModelT, NPROC, NQUEUE, NEVENT>>::type;

#ifdef CMB_HOST_BUILD
// the tier's source text run on the CPU (tests/cmb_engine_host.cpp): one trial, the slow path taken where it occurs
template <class Model, class S>
inline void static_run_trial_host(S &sim, Model &m, const TrialIn &in, TrialOut &out,
                                  uint64_t trace_cap, uint64_t *trace_key, double *trace_time)
{
    out.objects = 0u;
    out.sum_wait = 0.0;
    out.max_queue = 0u;
    for (int k = 0; k < 8; k++) out.counters[k] = 0u;
    m.run_trial(sim, in);
    if (!StaticKinds<Model>::agree(sim)) sim.status |= TRIAL_ERR_PROC_OVERFLOW;
    int who = 0;
    while (static_step(sim, m, who)) {
        if (sim.pops <= trace_cap) {
            trace_key[sim.pops - 1u] = sim.current_event;
            trace_time[sim.pops - 1u] = sim.now;
        }
        const uint32_t cmd = sim.cmd;
        sim.cmd = CMD_NONE;
        if (cmd == CMD_HOLD_EXPONENTIAL) {
            const double dur = gp_exponential(sim.rng, *sim.hot, sim.cmd_value);
            if (!sim.fel.schedule(who, ACT_WAKE_TIME, __dadd_rn(sim.now, dur), sim.prio_of((uint32_t)who))) sim.status |= TRIAL_ERR_FEL_OVERFLOW;
        }
        else if (cmd == CMD_HOLD_SAMPLED) {
            // as the device does it: the rectangles only first, and if they do not suffice the generator rewound and the whole sampler again
            const Sfc64 saved = sim.rng;
            const FlipState<S> saved_flips(sim);            // a sampler may call cmb_random_flip() before a draw gives up
            sim.hot_only = true;
            sim.hot_failed = false;
            double dur = ModelSampler<Model, S>::draw(m, sim, sim.cmd_sample);
            sim.hot_only = false;
            if (sim.hot_failed) {
                sim.hot_failed = false;
                sim.rng = saved;
                saved_flips.restore(sim);
                dur = ModelSampler<Model, S>::draw(m, sim, sim.cmd_sample);
            }
            if (dur < 0.0) sim.status |= TRIAL_ERR_NEGATIVE_HOLD;
            if (!sim.fel.schedule(who, ACT_WAKE_TIME, __dadd_rn(sim.now, dur), sim.prio_of((uint32_t)who))) sim.status |= TRIAL_ERR_FEL_OVERFLOW;
        }
        else {
            static_finish_command(sim, m, who, cmd);
        }
    }
    static_trial_end(sim);
    m.finish(sim, out);
}
#else

#ifndef STATIC_COLD_BATCH
#define STATIC_COLD_BATCH 4
#endif
#ifndef STATIC_PARK_MASK
#define STATIC_PARK_MASK 3u     // the parked set is examined every 4th step
#endif

// A model whose process bodies never draw themselves - every variate is the duration of a CMB_PROCESS_HOLD_EXPONENTIAL, drawn
// by the dispatcher - may say `static constexpr bool exponential_holds_only = true;`.  The dispatcher then keeps one raw sfc64
// output of look-ahead with its hot-path variate already formed (as mm1_fast.cuh does): the table look-up and the 64-bit ->
// double conversion leave the pop -> push chain.  The stream order is unchanged BECAUSE nothing else draws in between; a model
// with a cmb_random_* call in a body must not claim it.
template <class Model, class = void>
struct StaticLookahead {
    static constexpr bool value = false;
};
template <class Model>
struct StaticLookahead<Model, typename std::enable_if<Model::exponential_holds_only>::type> {
    static constexpr bool value = true;
};

// The kernel's launch bounds give ptxas 64 threads per CTA and, by default, no minimum of CTAs per SM: ptxas then picks a register
// target of its own, and for some models (coverage_models.cuh's PoolFightT, workshop_model.cuh's WorkshopT) that target is below
// what the step needs and it spills.  Such a model says `static constexpr int static_min_ctas = 1;`: one CTA per SM bounds the
// registers at 255 only, and ptxas allocates what the code needs.  0 (the default) leaves the bounds as they were.
template <class Model, class = void>
struct StaticMinCtas {
    static constexpr int value = 0;
};
template <class Model>
struct StaticMinCtas<Model, typename std::enable_if<(Model::static_min_ctas > 0)>::type> {
    static constexpr int value = Model::static_min_ctas;
};

struct StaticArgs {
    LaunchArgs base;
    double    *spill;           // [num_trials][NQUEUE][spill_cap]
    uint32_t   spill_cap;
};

template <template <class> class ModelT, int NPROC, int NQUEUE, int NEVENT, bool TRACE>
__global__ void __launch_bounds__(STATIC_BLOCK, StaticMinCtas<ModelT<StaticSim<NPROC, NQUEUE, NEVENT>>>::value)
static_trial_kernel(const StaticArgs sa)
{
    using S = StaticSimOf<ModelT, NPROC, NQUEUE, NEVENT>;
    __shared__ ZigHot hot;
    __shared__ double ring_smem[(NQUEUE > 0 ? NQUEUE : 1) * STATIC_WINDOW * STATIC_BLOCK];
    const LaunchArgs &a = sa.base;
    stage_zig_hot(hot, true);
    __syncthreads();

    constexpr unsigned FULL = 0xffffffffu;
    const uint64_t trial = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool alive = trial < a.num_trials;

    S sim;
    ModelT<S> m;
    TrialOut out;
    out.objects = 0u;
    out.sum_wait = 0.0;
    out.max_queue = 0u;
    for (int k = 0; k < 8; k++) out.counters[k] = 0u;
    sim.init(alive ? fmix64(a.master_seed, a.first_trial + trial) : 0u, &hot, &ring_smem[threadIdx.x], STATIC_BLOCK,
             (sa.spill_cap && alive) ? sa.spill + trial * (uint64_t)NQUEUE * sa.spill_cap : nullptr, sa.spill_cap);
    if (alive) {
        TrialIn in;
        in.arr_mean = a.arr_mean[trial];
        in.srv_mean = a.srv_mean[trial];
        in.num_objects = a.num_objects;
        in.servers = a.servers;
        in.num_params = a.num_params;
        for (int k = 0; k < 16; k++) in.params[k] = a.params[k];
        in.trial = a.first_trial + trial;
        m.run_trial(sim, in);
        if (!StaticKinds<ModelT<S>>::agree(sim)) sim.status |= TRIAL_ERR_PROC_OVERFLOW;
    }

#ifdef STATIC_NO_LOOKAHEAD
    constexpr bool AHEAD = false;
#else
    constexpr bool AHEAD = StaticLookahead<ModelT<S>>::value;
#endif
    bool parked = false;            // the exponential hold of this lane needs the ziggurat's slow path: wait for company
    uint64_t parked_u = 0u;
    int parked_who = 0;
    bool parked_sampled = false;    // ... or the sampler of its CMB_PROCESS_HOLD_SAMPLED does
    uint64_t u_next = 0u;           // AHEAD: the next raw output, drawn as soon as the previous one was consumed ...
    double e_next = 0.0;            // ... and its hot-path standard exponential
    if (AHEAD && alive) {
        u_next = sim.rng.next();
        e_next = Sfc64::exp_hot(hot, u_next);
    }
    uint32_t step = 0u;

    while (__any_sync(FULL, alive)) {
        bool draw = false, sampled = false;
        int who = 0;
        if (alive && !parked) {
            if (!static_step(sim, m, who)) {
                alive = false;                          // cmb_event_queue_execute returns
                static_trial_end(sim);
                m.finish(sim, out);
                if (a.events)    a.events[trial] = sim.pops;
                if (a.objects)   a.objects[trial] = out.objects;
                if (a.t_end)     a.t_end[trial] = sim.now;
                if (a.sum_wait)  a.sum_wait[trial] = out.sum_wait;
                if (a.status)    a.status[trial] = sim.status | (sim.fel.issued > 0x3ffffff0u ? TRIAL_ERR_KEY_OVERFLOW : 0u);
                if (a.max_queue) a.max_queue[trial] = out.max_queue;
                if (a.counters) {
                    for (int k = 0; k < 8; k++) a.counters[trial * 8u + k] = out.counters[k];
                }
            }
            else {
                if (TRACE) {
                    if (sim.pops <= a.trace_cap) {
                        a.trace_key[trial * a.trace_cap + sim.pops - 1u] = sim.current_event;
                        a.trace_time[trial * a.trace_cap + sim.pops - 1u] = sim.now;
                    }
                }
                const uint32_t cmd = sim.cmd;
                draw = cmd == CMD_HOLD_EXPONENTIAL;
                sampled = cmd == CMD_HOLD_SAMPLED;
                if (!draw && !sampled) static_finish_command(sim, m, who, cmd);
            }
        }
        // ---- converged: a sampled hold (CMB_PROCESS_HOLD_SAMPLED) - the model's sampler with the rectangles only; a lane whose
        // draw needs more rewinds the generator and parks
        if (sampled) {
            const Sfc64 saved = sim.rng;
            const FlipState<S> saved_flips(sim);            // a sampler may call cmb_random_flip() before a draw gives up
            sim.hot_only = true;
            sim.hot_failed = false;
            const double dur = ModelSampler<ModelT<S>, S>::draw(m, sim, sim.cmd_sample);
            sim.hot_only = false;
            if (sim.hot_failed) {
                sim.hot_failed = false;
                sim.rng = saved;
                saved_flips.restore(sim);
                parked = true;
                parked_sampled = true;
                parked_who = who;
            }
            else {
                if (dur < 0.0) sim.status |= TRIAL_ERR_NEGATIVE_HOLD;
                if (!sim.fel.schedule(who, ACT_WAKE_TIME, __dadd_rn(sim.now, dur), sim.prio_of((uint32_t)who))) sim.status |= TRIAL_ERR_FEL_OVERFLOW;
            }
        }
        // ---- converged: the hold's variate and its wake-up event (cmb_process_hold, src/cmb_process.c:262-285)
        if (draw) {
            const uint64_t u = AHEAD ? u_next : sim.rng.next();
            if (Sfc64::exp_is_hot(u)) {
                const double dur = __dmul_rn(sim.cmd_value, AHEAD ? e_next : Sfc64::exp_hot(hot, u));
                if (!sim.fel.schedule(who, ACT_WAKE_TIME, __dadd_rn(sim.now, dur), sim.prio_of((uint32_t)who))) sim.status |= TRIAL_ERR_FEL_OVERFLOW;
                if (AHEAD) {
                    u_next = sim.rng.next();
                    e_next = Sfc64::exp_hot(hot, u_next);
                }
            }
            else {
                parked = true;
                parked_u = u;
                parked_who = who;
            }
        }
        if ((++step & STATIC_PARK_MASK) != 0u) continue;
        const unsigned pm = __ballot_sync(FULL, parked);
        if (pm != 0u) {
            const unsigned am = __ballot_sync(FULL, alive);
            if (__popc(pm) >= STATIC_COLD_BATCH || pm == am) {
                if (parked) {
                    double dur;
                    if (parked_sampled) {
                        dur = ModelSampler<ModelT<S>, S>::draw(m, sim, sim.cmd_sample);
                        if (dur < 0.0) sim.status |= TRIAL_ERR_NEGATIVE_HOLD;
                    }
                    else {
                        dur = __dmul_rn(sim.cmd_value, sim.rng.exp_cold(parked_u));
                    }
                    if (!sim.fel.schedule(parked_who, ACT_WAKE_TIME, __dadd_rn(sim.now, dur), sim.prio_of((uint32_t)parked_who)))
                        sim.status |= TRIAL_ERR_FEL_OVERFLOW;
                    parked = false;
                    parked_sampled = false;
                    if (AHEAD) {
                        u_next = sim.rng.next();
                        e_next = Sfc64::exp_hot(hot, u_next);
                    }
                }
            }
        }
    }
}
#endif  // CMB_HOST_BUILD

}  // namespace cmb
}  // namespace cimba_b200
