// jtb_search.cuh — the throughput search kernel: ONE THREAD expands ONE configuration per CTA step.
//
// Same search as jtb_wgl.cuh (same keys, visited table, work ring, termination and pause/resume protocol — the two
// kernels are interchangeable behind jtb_check_linearizable), different mapping onto the SM:
//
//   jtb_wgl.cuh   a WARP expands one configuration, lane t evaluates open slot t.  Every child of a configuration is
//                 probed in the same round trip, which is what a latency-bound search wants (eager reads: ~1 new
//                 config per rank, 10k dependent ranks), but it costs ~550 warp instructions per configuration with
//                 half the lanes idle — instruction-bound.
//   this file     a THREAD expands one configuration (jtb_expand.h): candidate slots come from two bit masks in the
//                 frontier row, a bank read is rejected by one 32-bit hash compare, a transfer child needs no balance
//                 arithmetic until it turns out to be NEW (its balances are then patched in the queue entry), the
//                 frontier advance is a byte loop instead of match/ballot/redux rounds.  256 configurations per CTA
//                 step amortise the three barriers and thread 0's bookkeeping 8x better; 32 independent probe chains
//                 per warp keep the memory system busier than one.
//
// CTA step:  (A) barrier | thread 0: counters, donation, batch size, ring tickets | (B) barrier | donation copy,
//            ticket poll, batch claim (entry -> registers) | (C) barrier | expansion, children pushed on the CTA deque.
// Inside the expansion the threads of a warp run a warp-uniform loop "next consistent child of my configuration":
// one probe/insert per lane per round, then one warp-aggregated reservation on the CTA deque for the NEW children.
#pragma once
#include "jtb_expand.h"
#include "jtb_wgl.cuh"

namespace jtb {

#ifndef JTB_TPC_THREADS
#define JTB_TPC_THREADS 256
#endif
#ifndef JTB_TPC_CTAS
#define JTB_TPC_CTAS 3
#endif
constexpr int TPC_THREADS = JTB_TPC_THREADS;
constexpr int TPC_WARPS = TPC_THREADS / 32;
constexpr unsigned TPC_MAX_DONATE = TPC_THREADS;   // per step, when donating to hungry threads

struct TpcShared {
    int stop;
    unsigned top, bot;              // local LIFO deque (monotonic indices, masked on use)
    unsigned pop_top, don_bot;      // snapshots for this step's readers
    unsigned n_batch, n_don;
    unsigned n_holders;             // threads that hold a ring ticket
    unsigned assign_n, assign_next; // new tickets handed out this step, cursor over them
    unsigned n_exp, n_new;          // expansions / new children of the running step
    unsigned backoff;
    unsigned long long ticket_base, don_base;
    unsigned long long wit_cache;   // (shard << 32 | furthest rank): filter for the witness atomicMax
    unsigned long long polls;
    int since_flush;
};

template <int MODEL, int KW, bool EAGER>
__global__ void __launch_bounds__(TPC_THREADS, JTB_TPC_CTAS) wgl_tpc_kernel(const WglParams p, const int neg_ok) {
    using L = EntryLayout<MODEL, KW>;
    constexpr int EW = L::EW;
    constexpr unsigned FULL = 0xffffffffu;
    extern __shared__ __align__(16) uint64_t s_deque[];  // deque_cap * EW words
    __shared__ TpcShared sh;
    const int tid = threadIdx.x, lane = tid & 31;
    const unsigned lt_mask = (1u << lane) - 1;
    Ctrl* ctrl = p.ctrl;
    const unsigned cap_mask = p.deque_cap - 1;
    const unsigned high = p.deque_cap / 2;   // donate the oldest entries beyond this; overflow goes to the ring
    ExpandTables T;
    T.rows = p.rows; T.classes = p.classes; T.cls_inv_pos = p.cls_inv_pos; T.row_words = p.row_words; T.sum_off = 0;

    if (tid == 0) {
        sh.stop = 0; sh.top = sh.bot = 0;
        sh.n_holders = 0; sh.n_exp = 0; sh.n_new = 0;
        sh.backoff = 32;
        sh.wit_cache = ~0ull;
        sh.polls = 0; sh.since_flush = 0;
        const unsigned long long now = globaltimer();
        atomicCAS(&ctrl->t0, 0ull, now);
    }
    bool has_ticket = false;
    unsigned long long ticket = 0;
    unsigned long long my_configs = 0, my_probes = 0, my_expansions = 0;   // my_configs / my_expansions: lane 0
    int my_steps = 0, my_max_probe = 0;
    unsigned acc_new = 0, acc_exp = 0, acc_age = 0;  // thread 0 only
    int pre_stop = 0;                                // thread 0 only: control words read one step ahead
    unsigned long long pre_head = 0, pre_tail = 0;

    for (;;) {
        __syncthreads();  // (A) pushes of the previous step are complete
        if (tid == 0) {
            // ---- account the previous step (batched: only termination detection needs these) ---------
            acc_new += sh.n_new;
            acc_exp += sh.n_exp;
            const bool was_idle = sh.n_exp == 0;
            sh.n_exp = 0; sh.n_new = 0;
            int stop = pre_stop;
            const unsigned long long h = pre_head, t = pre_tail;   // prefetched during the last step
            const unsigned size = sh.top - sh.bot;
            // Invariant: an entry is counted in `created` before any other CTA can see it, and `created`
            // is always advanced before `expanded`.  So flush before donating, when idle, and periodically.
            const bool may_donate = stop == 2 || size > high || (h > t && size > (unsigned)TPC_THREADS);
            if ((acc_new | acc_exp) && (may_donate || (was_idle && size == 0) || ++acc_age >= 16)) {
                if (acc_new) { atomicAdd(&ctrl->created, (unsigned long long)acc_new); __threadfence(); }
                if (acc_exp) atomicAdd(&ctrl->expanded, (unsigned long long)acc_exp);
                acc_new = acc_exp = 0; acc_age = 0;
            }
            if (stop == 0) {
                if (t > h && t - h > p.ring_guard) {  // ring nearly full: pause (flush happens next step)
                    atomicCAS(&ctrl->cause, 0, CAUSE_RING_FULL);
                    atomicCAS(&ctrl->stop, 0, 2);
                }
                if (++sh.since_flush >= 64) {
                    sh.since_flush = 0;
                    if (p.time_budget_ns && globaltimer() - ld_volatile(&ctrl->t0) > p.time_budget_ns) {
                        atomicCAS(&ctrl->cause, 0, JTB_CAUSE_BUDGET);
                        atomicCAS(&ctrl->stop, 0, 2);
                    }
                }
                if (was_idle && size == 0) {
                    // nothing local, nothing served: termination test (expanded first, then created)
                    const unsigned long long ex = ld_volatile(&ctrl->expanded);
                    const unsigned long long cr = ld_volatile(&ctrl->created);
                    if (ex == cr) { atomicCAS(&ctrl->stop, 0, 1); stop = ld_volatile(&ctrl->stop); }
                    else {
                        stop = ld_volatile(&ctrl->stop);
                        __nanosleep(sh.backoff);
                        if (sh.backoff < 1024) sh.backoff <<= 1;
                    }
                } else {
                    sh.backoff = 32;
                }
            }
            sh.stop = stop;
            // ---- donation: deque nearly full, other threads hungry (tickets waiting), or pausing ---------
            const unsigned long long hunger = h > t ? h - t : 0;
            unsigned n_don = 0;
            if (stop == 2) n_don = size;  // pause: all live work must be in the ring
            else if (size > high) n_don = size - p.deque_cap / 4;
            else if (hunger && size > (unsigned)TPC_THREADS)
                n_don = (unsigned)min((unsigned long long)min(size - TPC_THREADS, TPC_MAX_DONATE), hunger);
            sh.n_don = n_don;
            sh.don_bot = sh.bot;
            if (n_don) {
                sh.don_base = atomicAdd(&ctrl->tail, (unsigned long long)n_don);
                sh.bot += n_don;
            }
            // ---- this step's batch: the deepest entries, one per thread -------------------------------------
            const unsigned n_batch = stop ? 0 : min(size - n_don, (unsigned)TPC_THREADS);
            sh.n_batch = n_batch;
            sh.pop_top = sh.top;
            sh.top -= n_batch;
            // fewer entries than threads: the surplus ticketless threads wait on ring tickets
            unsigned want = 0;
            if (!stop && n_batch + sh.n_holders < (unsigned)TPC_THREADS) want = TPC_THREADS - n_batch - sh.n_holders;
            sh.assign_n = want;
            sh.assign_next = 0;
            if (want) {
                sh.ticket_base = atomicAdd(&ctrl->head, (unsigned long long)want);
                sh.n_holders += want;
            }
        }
        __syncthreads();  // (B)
        if (sh.stop == 1) break;
        const bool exiting = sh.stop == 2;
        // ---- donation copy: oldest local entries -> ring (payload first, word0 = ready flag last) -----
        {
            const unsigned n_don = sh.n_don;
            for (unsigned i = tid; i < n_don; i += TPC_THREADS) {
                uint64_t* dst = p.ring + ((sh.don_base + i) & p.ring_mask) * EW;
                const uint64_t* src = &s_deque[(size_t)((sh.don_bot + i) & cap_mask) * EW];
                if (ld_volatile64(dst) != 0) atomicExch(&ctrl->overflow, 1);   // never overwrite live work silently
#pragma unroll
                for (int k = 1; k < EW; ++k) dst[k] = src[k];
                __threadfence();
                *(volatile uint64_t*)dst = src[0];
            }
        }
        Expander<MODEL, KW, EAGER> X;
        bool have = false;
        if (!exiting) {
            const unsigned n_batch = sh.n_batch;
            // ---- new ring tickets: only threads that have no batch entry this step take one ----------------
            if (sh.assign_n) {
                const unsigned wantm = __ballot_sync(FULL, !has_ticket && (unsigned)tid >= n_batch);
                unsigned base = 0;
                if (lane == 0 && wantm) base = atomicAdd(&sh.assign_next, (unsigned)__popc(wantm));
                base = __shfl_sync(FULL, base, 0);
                const unsigned mine = base + __popc(wantm & lt_mask);
                if (!has_ticket && (unsigned)tid >= n_batch && mine < sh.assign_n) {
                    ticket = sh.ticket_base + mine;
                    has_ticket = true;
                }
            }
            // ---- one poll of my ring ticket (a thread that owns a batch entry this step polls in a later step: an
            //      entry only ever has one owner, and a ticket stays valid until it is served) ------------------
            if (has_ticket && (unsigned)tid >= n_batch) {
                uint64_t* slot = p.ring + (ticket & p.ring_mask) * EW;
                const uint64_t w0 = ld_volatile64(slot);
                if (w0 != 0) {
                    __threadfence();  // acquire: payload words were written before word0
                    X.w[0] = w0;
#pragma unroll
                    for (int i = 1; i < KW; ++i) X.w[i] = ldcg64(slot + i);
                    if constexpr (L::HAS_BAL) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const uint64_t v = ldcg64(slot + KW + i);
                            X.bal[2 * i] = (int32_t)(uint32_t)v;
                            X.bal[2 * i + 1] = (int32_t)(uint32_t)(v >> 32);
                        }
                    }
                    __threadfence();  // the payload is in registers before the slot is released
                    *(volatile uint64_t*)slot = 0;
                    has_ticket = false;
                    have = true;
                }
            }
            const unsigned gotm = __ballot_sync(FULL, have);
            if (lane == 0) {
                if (gotm) atomicSub(&sh.n_holders, (unsigned)__popc(gotm));
                else if (tid == 0 && has_ticket) sh.polls++;
            }
            // ---- batch: thread t owns the t-th deepest local entry (every popped entry has exactly one owner) ----
            if ((unsigned)tid < n_batch) {
                const uint64_t* e = &s_deque[(size_t)((sh.pop_top - 1 - (unsigned)tid) & cap_mask) * EW];
#pragma unroll
                for (int i = 0; i < KW; ++i) X.w[i] = e[i];
                if constexpr (L::HAS_BAL) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint64_t v = e[KW + i];
                        X.bal[2 * i] = (int32_t)(uint32_t)v;
                        X.bal[2 * i + 1] = (int32_t)(uint32_t)(v >> 32);
                    }
                }
                have = true;
            }
        }
        __syncthreads();  // (C) entries are in registers, donated entries copied: pushes may reuse the space
        if (exiting) break;
        if (tid == 0) {  // prefetch the control words of the NEXT step behind this step's expansions
            pre_stop = ld_volatile(&ctrl->stop);
            pre_head = ld_volatile(&ctrl->head);
            pre_tail = ld_volatile(&ctrl->tail);
        }

        // ---------------- expansion --------------------------------------------------------------------
        unsigned n_new_total = 0, n_new_local = 0;   // warp-uniform
        // Space for the warp's `n` entries: on the CTA deque (returns false, `base` = first deque index) or, when the
        // deque is full, on the global ring (returns true, `rbase` = first ring position; `counted` entries are added
        // to `created` before they become visible).
        auto reserve = [&](unsigned n, bool counted, unsigned& base, unsigned long long& rbase) -> bool {
            int to_ring = 0;
            base = 0;
            rbase = 0;
            if (lane == 0) {
                unsigned old = *(volatile unsigned*)&sh.top;
                for (;;) {
                    if (old + n - sh.bot > p.deque_cap) { to_ring = 1; break; }
                    const unsigned seen = atomicCAS(&sh.top, old, old + n);
                    if (seen == old) { base = old; break; }
                    old = seen;
                }
                if (to_ring) {
                    if (counted) { atomicAdd(&ctrl->created, (unsigned long long)n); __threadfence(); }
                    rbase = atomicAdd(&ctrl->tail, (unsigned long long)n);
                }
            }
            base = __shfl_sync(FULL, base, 0);
            rbase = __shfl_sync(FULL, rbase, 0);
            return __shfl_sync(FULL, to_ring, 0) != 0;
        };
        // all lanes call push(); the NEW children of the warp get one reservation
        auto push = [&](bool is_new, const Child<KW>& ch) {
            const unsigned newm = __ballot_sync(FULL, is_new);
            if (newm == 0) return;
            const unsigned n = (unsigned)__popc(newm);
            unsigned base;
            unsigned long long rbase;
            const bool to_ring = reserve(n, true, base, rbase);
            const unsigned my = __popc(newm & lt_mask);
            if (!to_ring) {
                if (is_new) {
                    uint64_t* e = &s_deque[(size_t)((base + my) & cap_mask) * EW];
#pragma unroll
                    for (int i = 0; i < KW; ++i) e[i] = ch.w[i];
                    if constexpr (L::HAS_BAL) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) e[KW + i] = u64_of(X.bal[2 * i], X.bal[2 * i + 1]);
                        if (ch.amt) {   // the transfer that made this child: patch the two balances in place
                            int32_t* b32 = reinterpret_cast<int32_t*>(e + KW);
                            b32[ch.d] -= ch.amt;
                            b32[ch.c] += ch.amt;
                        }
                    }
                }
                n_new_local += n;
            } else if (is_new) {
                uint64_t* dst = p.ring + ((rbase + my) & p.ring_mask) * EW;
                if (ld_volatile64(dst) != 0) atomicExch(&ctrl->overflow, 1);   // never overwrite live work silently
#pragma unroll
                for (int i = 1; i < KW; ++i) dst[i] = ch.w[i];
                if constexpr (L::HAS_BAL) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int32_t lo = X.bal[2 * i] - (ch.d == 2 * i ? ch.amt : 0) + (ch.c == 2 * i ? ch.amt : 0);
                        const int32_t hi = X.bal[2 * i + 1] - (ch.d == 2 * i + 1 ? ch.amt : 0) +
                                           (ch.c == 2 * i + 1 ? ch.amt : 0);
                        dst[KW + i] = u64_of(lo, hi);
                    }
                }
                __threadfence();
                *(volatile uint64_t*)dst = ch.w[0];
            }
            n_new_total += n;
        };
        bool active = have;
        // a child that met a full table (rare: only around a table growth).  It was counted as a config when it was
        // queued; insert it now: already present -> un-count and drop, still full -> re-queue.
        {
            const bool retry = active && (X.w[0] & KEY_RETRY);
            if (__any_sync(FULL, retry)) {
                Child<KW> rq;
                bool requeue = false;
                if (retry) {
                    X.w[0] &= ~KEY_RETRY;
                    int plen;
                    const int res = table_insert_p<KW>(p, X.w, &plen);
                    if (res <= 0) {
                        active = false;
                        atomicAdd(&ctrl->configs, ~0ull);   // -1
                        if (res < 0) {
                            atomicCAS(&ctrl->cause, 0, JTB_CAUSE_TABLE_FULL);
                            atomicCAS(&ctrl->stop, 0, 2);
                            requeue = true;
                        }
                    }
                }
#pragma unroll
                for (int i = 0; i < KW; ++i) rq.w[i] = X.w[i];
                rq.w[0] |= KEY_RETRY;
                rq.amt = 0; rq.d = 0; rq.c = 0; rq.cgj = 0; rq.done = false;
                push(requeue, rq);
            }
        }
        X.todo = 0; X.rd_ok = 0; X.ncls = 0; X.cls_i = 0;
        if (active) {
            const int shard = X.load_header(T);
            const bool alive = !(p.n_shards > 1 && ld_volatile(&p.shard_found[shard]));
            X.begin(T, alive);
        }
        for (;;) {
            Child<KW> ch;
            const bool hc = active && X.next(T, neg_ok != 0, ch);
            if (!__any_sync(FULL, hc)) break;
            bool is_new = false;
            if (hc) {
                if (ch.done) {
                    // every :ok op of the shard is linearized -> VALID
                    if (atomicExch(&p.shard_found[X.shard], 1) == 0) {
                        if (atomicSub(&ctrl->n_undecided, 1) == 1) atomicCAS(&ctrl->stop, 0, 1);
                    }
                } else {
                    int plen;
                    const int res = table_insert_p<KW>(p, ch.w, &plen);
                    my_probes++;
                    my_max_probe = max(my_max_probe, plen);
                    if (res < 0) {
                        // table exhausted: pause for growth; the child is queued un-inserted (KEY_RETRY)
                        atomicCAS(&ctrl->cause, 0, JTB_CAUSE_TABLE_FULL);
                        atomicCAS(&ctrl->stop, 0, 2);
                        ch.w[0] |= KEY_RETRY;
                    }
                    is_new = res != 0;
                    if (is_new && ch.cgj > X.gj) {
                        // witness bookkeeping: furthest frontier reached in this shard
                        const unsigned long long wc = *(volatile unsigned long long*)&sh.wit_cache;
                        if ((int)(wc >> 32) != X.shard || (int)(uint32_t)wc < ch.cgj) {
                            *(volatile unsigned long long*)&sh.wit_cache =
                                ((unsigned long long)(uint32_t)X.shard << 32) | (uint32_t)ch.cgj;
                            atomicMax(&p.shard_max_rank[X.shard], ch.cgj);
                        }
                    }
                }
            }
            push(is_new, ch);
        }
        const unsigned expm = __ballot_sync(FULL, have);
        if (lane == 0) {
            if (n_new_local) atomicAdd(&sh.n_new, n_new_local);
            if (expm) atomicAdd(&sh.n_exp, (unsigned)__popc(expm));
            my_expansions += __popc(expm);
            my_configs += n_new_total;
            if (++my_steps >= 8 || my_configs >= 2048) {
                // amortised global tally: budget (max_configs) and table-load guard
                my_steps = 0;
                if (my_configs) {
                    const unsigned long long tot = atomicAdd(&ctrl->configs, my_configs) + my_configs;
                    my_configs = 0;
                    if (tot >= p.max_configs) {
                        atomicCAS(&ctrl->cause, 0, p.budget_cause);
                        atomicCAS(&ctrl->stop, 0, 2);
                    }
                }
            }
        }
    }
    // ---- flush statistics -------------------------------------------------------------------------
    for (int o = 16; o > 0; o >>= 1) {
        my_probes += __shfl_xor_sync(FULL, my_probes, o);
        my_max_probe = max(my_max_probe, __shfl_xor_sync(FULL, my_max_probe, o));
    }
    if (lane == 0) {
        atomicAdd(&ctrl->configs, my_configs);
        atomicAdd(&ctrl->probes, my_probes);
        atomicAdd(&ctrl->expansions, my_expansions);
        atomicMax(&ctrl->max_probe_len, (unsigned long long)my_max_probe);
    }
    if (tid == 0) atomicAdd(&ctrl->polls, sh.polls);
}

}  // namespace jtb
