// mm1_fast.cuh - the M/M/1 replication kernel, written for SIMT issue efficiency.
//
// Same model, same per-trial arithmetic and the same order of random draws, key
// issues and pops as queue_kernel<0> in queue_model.cuh (which stays as the
// readable formulation and serves G/G/1); see that file for the mapping onto
// benchmark/MM1_multi.c:52-125 and the reference's dispatcher.
//
// What is different is only how a warp executes it.  In queue_kernel<0> the
// arrival and service process bodies are separate divergent regions wrapped in
// reconvergence barriers, and many of the issued instructions are register moves
// merging those regions' results.  With few warps per scheduler the kernel is
// bound by dependent-issue latency.  Here one event step is a single
// straight-line, predicated sequence that all 32 lanes execute together:
//   the pop of the first of the two pending events, which are kept in time
//   order, the arrival body and the service body as predicated updates of the
//   same registers (a lane is in exactly one of them), the variate draw and the
//   wake-up insert (one compare and selects).  The only branches left are the
//   look-ahead refill and the rare ones: queue spill to HBM, trial completion
//   and the parked ziggurat slow path.
#pragma once

#include "engine.cuh"
#include "queue_model.cuh"
#include "rng.cuh"

namespace cimba_b200 {

// tuning knobs
#ifndef MM1_PARK_MASK
#define MM1_PARK_MASK 7u      // the parked set is examined every 8th step
#endif
#ifndef MM1_COLD_BATCH
#define MM1_COLD_BATCH 4       // parked lanes needed before the ziggurat slow path runs
#endif
#ifndef MM1_STEPS
#define MM1_STEPS 8            // event steps per loop iteration (a multiple or a divisor of MM1_PARK_MASK + 1)
#endif

// Shared-memory ring entries per trial.  A take that leaves more than this many waiting refills the freed slot from the
// trial's HBM ring, a round trip the whole warp waits for; at rho = 0.9 a queue passes 48 about 1 / 0.9^16 = 5.4 times
// less often than it passes 32.  The ring (one row of QUEUE_BLOCK doubles per entry), the row that takes the stores of
// lanes that do not put, and the ziggurat table come to 27 136 B: 8 CTAs + the 1 KB the hardware reserves per CTA fit the
// 228 KB an SM has when the kernel asks for the largest shared-memory carveout (capi.cu does).
constexpr int MM1_WINDOW = 48;
static_assert(8 * ((MM1_WINDOW + 1) * QUEUE_BLOCK * 8 + 256 * 8 + 1024) <= 228 * 1024,
              "8 CTAs of mm1_kernel must fit an SM: 65 536 trials in one wave on 132 SMs");

// 32-bit shared-window accesses: one address register, no generic->shared
// conversion per access (the static-__shared__ form costs extra
// instructions each time).
__device__ __forceinline__ void sts_f64(uint32_t addr, double v)
{
    asm volatile("st.shared.f64 [%0], %1;" :: "r"(addr), "d"(v) : "memory");
}

__device__ __forceinline__ double lds_f64(uint32_t addr)
{
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory");
    return v;
}

// Event keys carry the action in their two low bits: key = (issue counter << 2) | action.
// Counters are unique, so ordering by this word is ordering by issue counter (the
// reference's FIFO tie-break, src/cmi_hashheap.c:55-80) and one register holds both.
// A key issued later is the larger, as long as the counter stays below 2^30.
__device__ __forceinline__ uint32_t pack_key(uint32_t counter, uint32_t action)
{
    return (counter << 2) | action;
}

template <bool TRACE>
__global__ void __launch_bounds__(QUEUE_BLOCK)
mm1_kernel(const QueueArgs a)
{
    __shared__ double exp_x[256];                       // ziggurat layer widths (hot table)
    __shared__ double ring_smem[(MM1_WINDOW + 1) * QUEUE_BLOCK];   // MM1_WINDOW rows of ring, then the scratch row

    for (unsigned i = threadIdx.x; i < 256u; i += blockDim.x) {
        exp_x[i] = zig::zig_exp_x[i];
    }
    __syncthreads();

    constexpr unsigned FULL = 0xffffffffu;
    constexpr uint32_t ROW = QUEUE_BLOCK * 8u;          // bytes between consecutive ring entries of one trial
    const double INF = __longlong_as_double(0x7ff0000000000000LL);
    const unsigned lane = threadIdx.x & 31u;
    const uint64_t gtid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t trial;
    bool alive;
    if (a.mapping == 32) {
        trial = gtid >> 5;
        alive = (lane == 0u) && (trial < a.num_trials);
    }
    else {
        trial = gtid;
        alive = trial < a.num_trials;
    }

    // ---- per-trial state (registers)
    Sfc64 rng;
    rng.a = rng.b = rng.c = rng.d = 0u;
    // The two pending events in pop order: slot 0 is the next to pop, slot 1 the other.  Each process owns at most one
    // pending event, so the two slots belong to different processes, and one word says which: slot 0 is the arrival
    // process's when `lead_arr` is 1, the service process's when it is 0.  An empty slot has time +inf and key 0 (action
    // ACT_NONE) and belongs to the process that has no event pending.
    double t0 = INF, t1 = INF;
    uint32_t k0 = 0u, k1 = 0u;
    uint32_t lead_arr = 1u;
    // item_counter (src/cmi_hashheap.c:449-453) kept as the WAKE_TIME key of the last counter issued,
    // (counter << 2) | ACT_WAKE_TIME, so that issuing a key is one add of 4.  The word wraps when the counter reaches
    // 2^30, as the keys do; `wraps` counts that (once per loop iteration, which issues far fewer than 2^30 keys), so the
    // event count written after the loop is exact.
    uint32_t last_key = ACT_WAKE_TIME, last_seen = ACT_WAKE_TIME, wraps = 0u;
    double now = 0.0, stamp = 0.0, sum_wait = 0.0;
    double arr_mean = 1.0, srv_mean = 1.0;
    // FIFO discipline: the k-th object put is the k-th object taken, so the ring's
    // tail index is `produced`, its head index is `served`, its length their difference.
    // The server is waiting at the front guard exactly when no other event is pending
    // at the moment an arrival puts (it otherwise always owns one pending event).
    uint32_t produced = 0u, served = 0u, dropped = 0u, status = TRIAL_OK, longest = 0u;
    const uint32_t quota = (uint32_t)a.num_objects;
    // The window's tail and head slots (`produced` and `served` modulo MM1_WINDOW) as byte offsets from the ring's start,
    // the lane's column included, advanced wherever the counters are.  Every offset stays in the ring, a void trial's too.
    const uint32_t ring = (uint32_t)__cvta_generic_to_shared(&ring_smem[0]);
    uint32_t tail = threadIdx.x * 8u, head = threadIdx.x * 8u;
    const uint32_t scratch = MM1_WINDOW * ROW + threadIdx.x * 8u;   // sink for the store of lanes that do not put
    // the next slot: off + ROW, or back to the first row from the last, where off + ROW - MM1_WINDOW * ROW is the smaller
    // (below the last row it wraps past 2^32)
    const auto next_slot = [](uint32_t off) { return min(off + ROW, off - (MM1_WINDOW - 1) * ROW); };
    uint32_t tab = (uint32_t)__cvta_generic_to_shared(&exp_x[0]);
    asm volatile("" : "+r"(tab));                       // keep in a register (no per-step rematerialisation)
    double *const spill = (a.spill_cap && alive) ? a.spill + trial * a.spill_cap : nullptr;
    const uint32_t spill_mask = a.spill_cap - 1u;

    // one variate of look-ahead: the next raw sfc64 output is drawn as soon as the
    // previous one is consumed, so its table lookup and conversion are off the
    // critical path of the step that uses it.  The stream order is unchanged; one
    // unused raw draw remains when the trial ends.
    uint64_t u_next = 0u;
    double e_next = 0.0;                                // hot-path std exponential of u_next
    uint32_t off_next = 0u;                             // u_next's ziggurat layer as a byte offset into exp_x
    uint32_t pops = 0u;
    // (u & 0xff) * 8 as hi((u << 24) * 2^11): two IMADs instead of a shift and a mask
    const auto refill = [&]() {
        u_next = rng.next_imad();
        off_next = imad_hi(imad_lo((uint32_t)u_next, IMAD_K2P24, 0u), IMAD_K2P11, 0u);
        e_next = __dmul_rn(lds_f64(tab + off_next), __ull2double_rn(u_next));
    };

    if (alive) {
        arr_mean = a.arr_mean[trial];
        srv_mean = a.srv_mean[trial];
        rng.seed(fmix64(a.master_seed, a.first_trial + trial));
        t0 = 0.0; k0 = pack_key(1u, ACT_START);         // cmb_process_start(arrival), MM1_multi.c:107-108
        t1 = 0.0; k1 = pack_key(2u, ACT_START);         // cmb_process_start(service), :109-111
        last_key = last_seen = pack_key(2u, ACT_WAKE_TIME);
        refill();
    }

    // lane state in one word: 1 running, 3 parked (the look-ahead variate needs the ziggurat
    // slow path) in the service process, 7 parked in the arrival process, 0 finished
    uint32_t flags = alive ? 1u : 0u;
    uint32_t step = 0u;

    // One event step.  A lane that is finished or parked runs it with every update predicated off, so the registers of a
    // finished trial hold its results until they are written after the loop.
    const auto event_step = [&]() {
        // ---------------- pop (cmi_hashheap_dequeue order: time asc, key asc): slot 0
        const bool go0 = flags == 1u;                   // alive and not parked
        const uint32_t key = k0;
        const bool go = go0 & (key != 0u);
        if (go0 & (key == 0u)) flags = 0u;              // event list ran dry: the trial is over
        const bool is_arr = go & (lead_arr != 0u);
        const bool is_srv = go & (lead_arr == 0u);
        const bool wake = (key & 3u) == ACT_WAKE_TIME;
        if (TRACE) {
            if (go && pops < a.trace_cap) {
                a.trace_key[trial * a.trace_cap + pops] = key >> 2;
                a.trace_time[trial * a.trace_cap + pops] = t0;
            }
            pops += go ? 1u : 0u;
        }
        if (go) now = t0;                               // src/cmb_event.c:239-241

        // ---------------- arrival body (MM1_multi.c:58-66): back from hold -> put
        // Ring accesses are unconditional (a lane that does not put writes its private
        // scratch row instead): a select on the address is cheaper than a divergent region.
        const uint32_t p0 = produced, s0 = served;
        const uint32_t q_len = p0 - s0;
        const bool put = is_arr & wake;
        const bool put_far = put & (q_len >= (uint32_t)MM1_WINDOW);
        sts_f64(ring + ((put & !put_far) ? tail : scratch), now);
        if (put) {
            produced++;
            tail = next_slot(tail);
        }
        // cmb_objectqueue_put -> cmb_resourceguard_signal(front guard): wake the server.  The arrival process popped, so
        // slot 1 is the server's, and it is empty exactly when the server waits at the front guard.
        if (put & (k1 == 0u)) {
            last_key += 4u;
            t1 = now;
            k1 = last_key | ACT_WAKE_RESOURCE;
        }

        // ---------------- service body (MM1_multi.c:78-88)
        const double new_sum = __dadd_rn(sum_wait, __dsub_rn(now, stamp));
        if (is_srv & wake) sum_wait = new_sum;          // back from the service hold
        // cmb_objectqueue_get: take the head, or wait at the front guard (slot stays empty)
        const bool take = is_srv & (q_len != 0u);
        const uint32_t h0 = head;
        const double head_stamp = lds_f64(ring + h0);   // harmless when the ring is empty
        if (take) {
            stamp = head_stamp;
            served++;
            head = next_slot(head);
        }
        const bool refill_far = take & (q_len > (uint32_t)MM1_WINDOW);

        // ---------------- hold: consume the look-ahead variate, insert the wake-up
        const bool draw = take | (is_arr & (produced < quota));
        const bool hot = off_next <= ZIG_EXP_MAX * 8u;  // Sfc64::exp_is_hot(u_next)
        const bool push = draw & hot;
        const double when = __dadd_rn(now, __dmul_rn(is_arr ? arr_mean : srv_mean, e_next));
        if (push) last_key += 4u;
        const uint32_t k_new = last_key;
        // The popped process's next event, if it has one, goes in beside the other pending event (slot 1, the server's
        // wake-up above included).  Its key is the largest issued so far, so on a tie in time the other goes first, and one
        // strict compare orders the pair.  A lane that pops either puts its new event ahead or swaps the other one to the
        // front (with its new event, or none, behind); a lane that does not pop does neither.
        const bool ahead = push & (when < t1);
        const bool swap = go & !ahead;
        const double t_lead = swap ? t1 : (push ? when : t0);
        const uint32_t k_lead = swap ? k1 : (push ? k_new : k0);
        if (swap) {
            t1 = push ? when : INF;
            k1 = push ? k_new : 0u;
            lead_arr ^= 1u;                             // the other process leads now
        }
        t0 = t_lead;
        k0 = k_lead;
        if (draw & !hot) flags = is_arr ? 7u : 3u;
        if (push) refill();

        // ---------------- rare: the queue reaches past the on-chip window
        if (put_far | refill_far) {
            if (refill_far) {                           // refill the freed slot from HBM
                sts_f64(ring + h0, spill[(s0 + MM1_WINDOW) & spill_mask]);
            }
            else if (spill != nullptr && q_len - MM1_WINDOW <= spill_mask) {
                spill[p0 & spill_mask] = now;
            }
            else {
                status |= TRIAL_ERR_QUEUE_OVERFLOW;     // entry dropped: the trial is void from here on
                dropped++;
                served++;                               // keep produced - served = entries actually stored
                head = next_slot(head);
            }
        }
        longest = max(longest, produced - served);
    };

    // MM1_STEPS event steps per iteration share one exit vote and one look at the parked set.  Eight (one whole parked-set
    // period) unrolled leave ptxas the most room to overlap the steps' independent work: 6 % faster than 2 (H100 SXM, 700 W).
    while (__any_sync(FULL, flags & 1u)) {
#pragma unroll
        for (int i = 0; i < MM1_STEPS; i++) {
            event_step();
        }
        step += MM1_STEPS;
        wraps += last_key < last_seen ? 1u : 0u;
        last_seen = last_key;
        if ((step & MM1_PARK_MASK) != 0u) {
            continue;                                   // look at the parked set every (MM1_PARK_MASK+1)-th step only
        }
        const unsigned pm = __ballot_sync(FULL, flags & 2u);
        if (pm != 0u) {
            const unsigned am = __ballot_sync(FULL, flags & 1u);
            if (__popc(pm) >= MM1_COLD_BATCH || pm == am) {
                if (flags & 2u) {
                    const bool parked_is_arr = (flags & 4u) != 0u;
                    const double mean = parked_is_arr ? arr_mean : srv_mean;
                    const double at = __dadd_rn(now, __dmul_rn(mean, rng.exp_cold(u_next)));
                    last_key += 4u;
                    const uint32_t k_at = last_key;
                    // the parking step left the other process's event (or none) in slot 0 and slot 1 empty: insert
                    // beside slot 0 as an event step inserts beside slot 1
                    const bool first = at < t0;
                    t1 = first ? t0 : at;
                    k1 = first ? k0 : k_at;
                    t0 = first ? at : t0;
                    k0 = first ? k_at : k0;
                    lead_arr = (first == parked_is_arr) ? 1u : 0u;
                    flags = 1u;
                    refill();
                }
            }
        }
    }
    // every update above is predicated on a running lane: the registers hold each trial's results
    const uint32_t issued = (wraps << 30) + (last_key >> 2);
    if (alive) {
        if (a.events)    a.events[trial] = issued;      // every scheduled event has been popped
        if (a.objects)   a.objects[trial] = served - dropped;
        if (a.t_end)     a.t_end[trial] = now;
        if (a.sum_wait)  a.sum_wait[trial] = sum_wait;
        if (a.status)    a.status[trial] = status | (issued > 0x3ffffff0u ? TRIAL_ERR_KEY_OVERFLOW : 0u);
        if (a.max_queue) a.max_queue[trial] = longest;
    }
    if (a.diag != nullptr && lane == 0u) {             // bench.py: event steps -> issued warp-instructions
        atomicAdd(a.diag, (unsigned long long)step);
        atomicAdd(a.diag + 1, 1ull);
    }
}

}  // namespace cimba_b200
