// jtb_wgl.cuh — Wing–Gong/Lowe linearizability search as a persistent sm_90a kernel.
//
// Replaces the hot loop of knossos.wgl/analysis behind jepsen.checker/linearizable (SURVEY.md §3.3,
// A.5): `cache.add((linearized BitSet, model))` + `model.step`.  GPU-first formulation:
//
//  * A configuration is keyed EXACTLY by its window form
//        word0 = valid | global return rank of the first un-linearized :ok op | register state
//        word1 = bitmask over the (<=64) open-op slots at that return  + crashed-class counts
//        word2.. = more crashed-class counts (KW = 2, 4 or 8 words)
//    (every op that returned earlier is necessarily linearized; crashed ops of one (f, value) class
//    are consumed in invocation order so a count identifies the consumed set).
//  * One warp expands one configuration per step: lane t evaluates the op in open slot t
//    (model step inlined), the lane that linearizes the frontier op advances the frontier with
//    ballot/match arithmetic, every consistent child is probed/inserted in the global visited table
//    (16 B slots, ld.global.cg.v2.u64 probe + atom.cas.b128 insert), new children are pushed on the
//    CTA's shared-memory staging buffer.
//  * Work distribution: depth-first locally, breadth-first globally, no locks.
//      - each CTA keeps a LIFO deque in shared memory shared by its 8 warps (deep dives find the
//        linearization of a valid history quickly).  A barrier-free variant with one private deque per
//        warp was also measured: correct, but slower (private stacks fragment the work: many more idle
//        polls) even though bar.sync is the top stall reason of this version;
//      - an idle warp takes a read TICKET (ring position from atomicAdd(head)) on a global FIFO ring in HBM
//        and polls that slot; head - tail > 0 is therefore the number of hungry warps;
//      - a CTA whose deque is nearly full, or that sees hungry warps, donates its OLDEST entries with one
//        atomicAdd(tail) (payload words first, word0 = ready flag last); the ticket holder zeroes the slot.
//    A lock-based LIFO pool with stealing was measured first and starved (46 M idle spins for 4.8 M
//    configs); a pure FIFO was 50x faster on exhaustive searches but explodes on valid histories with
//    crashed ops (breadth-first visits the whole reachable space).  This hybrid keeps both properties.
//    Termination: expanded == created.  Pause/resume: on pause every CTA flushes its deque, so the live
//    work is exactly the non-zero ring slots and the host can grow the table or the ring and relaunch.
//  * Verdict: first config whose frontier passes the shard's last return => VALID (early exit);
//    exhaustion => INVALID with witness = furthest frontier rank reached (atomicMax), which is the
//    earliest :ok completion whose history prefix is not linearizable (SURVEY §7.4-5).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "jtb_prep.h"

namespace jtb {

struct __align__(16) K128 {
    uint64_t lo, hi;
};

struct Ctrl {
    // each hot word on its own 128 B line (same-line atomics serialise in one L2 slice)
    alignas(128) int stop;         // 0 run, 1 finished (all shards decided or exhausted), 2 paused/aborted (cause)
    int cause;                     // JTB_CAUSE_* / CAUSE_RING_FULL when stop == 2
    int n_undecided;               // shards not yet found VALID
    int overflow;                  // a ring slot was overwritten before it was consumed: the verdict is void (UNKNOWN)
    alignas(128) unsigned long long head;   // read tickets handed to warps (ring positions)
    alignas(128) unsigned long long tail;   // entries pushed (ring positions reserved for writing)
    alignas(128) unsigned long long created;   // configs created (initial + every new child)
    alignas(128) unsigned long long expanded;  // configs expanded; created == expanded <=> search exhausted
    alignas(128) unsigned long long configs;  // distinct configs inserted (amortised tally; budget / load guard)
    alignas(128) unsigned long long t0;       // %globaltimer at first CTA start
    unsigned long long probes, expansions, polls, max_probe_len, max_live;
};
constexpr int CAUSE_RING_FULL = 100;  // internal: the host grows the ring and resumes

struct WglParams {
    const int32_t* rows;        // frontier rows with the slot ops inline (jtb_prep.h)
    const ClassRec* classes;
    const int32_t* cls_inv_pos;
    uint64_t* table;        // slots of KW 64-bit words
    uint64_t slot_mask;     // n_slots - 1
    uint64_t* ring;         // work queue: entries of EW words, word0 != 0 <=> slot holds an entry
    uint64_t ring_mask;     // ring entries - 1
    uint64_t ring_guard;    // pause when (tail - head) exceeds this
    Ctrl* ctrl;
    int* shard_found;       // [n_shards]
    int* shard_max_rank;    // [n_shards] furthest frontier reached (global rank)
    int row_words, S_pad, n_shards, max_nc;
    unsigned long long max_configs;   // stop (UNKNOWN) once this many configs were inserted
    int budget_cause;                 // JTB_CAUSE_BUDGET or JTB_CAUSE_TABLE_FULL (load guard)
    unsigned long long time_budget_ns;
    uint32_t deque_cap;     // entries in the CTA's shared-memory deque (power of two)
    int eager_reads;        // linearize a consistent candidate read immediately and exclusively
};

constexpr uint64_t KEY_VALID = 1ull << 63;
constexpr uint64_t KEY_LOCK = 1ull << 62;   // only used by KW > 2 slots while their tail is written
// Queue entries only (never stored in the table): the config could not be inserted because its probe sequence ran
// off a full table; whoever pops it inserts it first (after the host has grown the table) — no work is lost.
constexpr uint64_t KEY_RETRY = 1ull << 61;
constexpr uint32_t RANK_MASK = 0x1fffffffu;  // global return rank: bits 32..60 of word 0
constexpr int MAX_PROBE = 512;

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ K128 ldcg128(const void* p) {
    K128 r;
    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(r.lo), "=l"(r.hi) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ uint64_t ldcg64(const void* p) {
    uint64_t r;
    asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(r) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ K128 cas128(void* addr, K128 cmp, K128 val) {
    K128 old;
    asm volatile(
        "{\n\t"
        ".reg .b128 c, v, o;\n\t"
        "mov.b128 c, {%2, %3};\n\t"
        "mov.b128 v, {%4, %5};\n\t"
        "atom.relaxed.gpu.global.cas.b128 o, [%6], c, v;\n\t"
        "mov.b128 {%0, %1}, o;\n\t"
        "}\n"
        : "=l"(old.lo), "=l"(old.hi)
        : "l"(cmp.lo), "l"(cmp.hi), "l"(val.lo), "l"(val.hi), "l"(addr)
        : "memory");
    return old;
}
__device__ __forceinline__ int ld_volatile(const int* p) { return *(const volatile int*)p; }
__device__ __forceinline__ unsigned long long ld_volatile(const unsigned long long* p) {
    return *(const volatile unsigned long long*)p;
}
__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

template <int KW>
__device__ __forceinline__ uint64_t hash_key(const uint64_t (&k)[KW]) {
    uint64_t h = mix64(k[0] ^ 0x9E3779B97F4A7C15ull);
#pragma unroll
    for (int i = 1; i < KW; ++i) h = mix64(h ^ k[i] + 0x9E3779B97F4A7C15ull * (uint64_t)(i + 1));
    return h;
}

// Visited-table probe + insert.  Returns 1 = inserted (new config), 0 = already present,
// -1 = table exhausted.  *plen gets the number of slots inspected.  Linear probing from hash & slot_mask.
template <int KW>
__device__ __forceinline__ int table_insert(uint64_t* table, uint64_t slot_mask, const uint64_t (&k)[KW], int* plen,
                                            bool cas_first = false) {
    uint64_t idx = hash_key<KW>(k) & slot_mask;
    for (int i = 0; i < MAX_PROBE; ++i) {
        uint64_t* slot = table + idx * KW;
        // load-first: hits (the majority) cost one plain load; cas-first: new configs cost one round trip
        K128 cur = (KW == 2 && cas_first) ? K128{0, 0} : ldcg128(slot);
        if (cur.lo == 0 && cur.hi == 0) {
            K128 mine{KW == 2 ? k[0] : (k[0] | KEY_LOCK), k[1]};
            K128 old = cas128(slot, K128{0, 0}, mine);
            if (old.lo == 0 && old.hi == 0) {
                if constexpr (KW > 2) {
#pragma unroll
                    for (int w = 2; w < KW; ++w) slot[w] = k[w];
                    __threadfence();
                    *(volatile uint64_t*)slot = k[0];  // unlock
                }
                *plen = i + 1;
                return 1;
            }
            cur = old;
        }
        if constexpr (KW == 2) {
            if (cur.lo == k[0] && cur.hi == k[1]) { *plen = i + 1; return 0; }
        } else {
            if ((cur.lo & ~KEY_LOCK) == k[0] && cur.hi == k[1]) {
                while (cur.lo & KEY_LOCK) cur.lo = ldcg64(slot);
                __threadfence();
                bool same = true;
#pragma unroll
                for (int w = 2; w < KW; ++w) same &= ldcg64(slot + w) == k[w];
                if (same) { *plen = i + 1; return 0; }
            }
        }
        idx = (idx + 1) & slot_mask;
    }
    *plen = MAX_PROBE;
    return -1;
}

// ------------------------------------------------------------------------------------------------
// Model step, inlined per lane (knossos.model, SURVEY A.4; bank: SURVEY §8(a) A7 from
// src/tigerbeetle/tests/ledger.clj:89-152).  `reg` is the register value (word0 low half),
// `bal` the 8 balances carried in the entry.
// `cell` points at the op's inline record in the frontier row (OpRec, then the model's read payload).
template <int MODEL>
__device__ __forceinline__ bool model_step(const int4 op, int32_t& reg, int32_t (&bal)[8],
                                           const int32_t* __restrict__ cell, bool neg_ok, uint64_t w1) {
    const int f = op.x & 0xff;
    if (op.x & OP_IMPOSSIBLE) return false;
    if constexpr (MODEL == JTB_MODEL_REGISTER || MODEL == JTB_MODEL_CAS_REGISTER) {
        if (f == JTB_F_READ) return op.y == JTB_NIL || op.y == reg;
        if (f == JTB_F_WRITE) { reg = op.y; return true; }
        if (reg != op.y) return false;  // cas
        reg = op.z;
        return true;
    } else if constexpr (MODEL == JTB_MODEL_BANK) {
        if (f == JTB_F_TRANSFER) {
            bool ok = true;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (i == op.z) { bal[i] -= op.y; ok &= neg_ok || bal[i] >= 0; }
                if (i == op.w) bal[i] += op.y;
            }
            return ok;
        }
        // read: every account present in the payload must match
        const int4* rb = reinterpret_cast<const int4*>(cell + 4);
        const int4 lo = __ldg(rb), hi = __ldg(rb + 1);
        const int care = op.y;
        bool ok = true;
        ok &= !(care & 1) || bal[0] == lo.x;
        ok &= !(care & 2) || bal[1] == lo.y;
        ok &= !(care & 4) || bal[2] == lo.z;
        ok &= !(care & 8) || bal[3] == lo.w;
        ok &= !(care & 16) || bal[4] == hi.x;
        ok &= !(care & 32) || bal[5] == hi.y;
        ok &= !(care & 64) || bal[6] == hi.z;
        ok &= !(care & 128) || bal[7] == hi.w;
        return ok;
    } else if constexpr (MODEL == JTB_MODEL_SET) {
        // grow-only set: adds always apply; a read is consistent iff the constrained bits of key word 1
        // (open-slot mask + crashed-add counts) equal the precomputed pattern for this (read, frontier)
        if (f == JTB_F_ADD) return true;
        const ulonglong2 nc = __ldg(reinterpret_cast<const ulonglong2*>(cell + 4));
        return (w1 & nc.y) == nc.x;
    } else {
        return false;
    }
}

// One expansion, warp-synchronous: evaluates every candidate of the configuration (w, pbal), probes/inserts the
// consistent children and hands the NEW ones to `push(is_new, key words, balances)` (called by all lanes, once per
// candidate round).  Shared by the search kernels; `wit_cache` is a shared-memory filter for the witness atomicMax.
template <int MODEL, int KW, bool EAGER, typename Push>
__device__ __forceinline__ void expand_config(const WglParams& p, Ctrl* ctrl, const int neg_ok, const uint64_t (&w)[KW],
                                              const int32_t (&pbal)[8], const int lane, unsigned long long* wit_cache, unsigned long long& my_probes,
                                              int& my_max_probe, Push&& push) {
    constexpr int SW = MODEL == JTB_MODEL_BANK ? 12 : MODEL == JTB_MODEL_SET ? 8 : 4;  // = slot_words(MODEL)
    const int cand_rounds = p.S_pad / 32;
    const int cls_rounds = (p.max_nc + 31) / 32;
    const int gj = (int)((w[0] >> 32) & RANK_MASK);
    const int32_t preg = (int32_t)(uint32_t)w[0];
    const int32_t* row = p.rows + (size_t)gj * p.row_words;
    const int32_t extra = __ldg(row + (lane & 15));
    const int fr_pos = __shfl_sync(0xffffffffu, extra, 8);
    const int shard = __shfl_sync(0xffffffffu, extra, 9);
    const int gj_end = __shfl_sync(0xffffffffu, extra, 10);
    const int cls_base = __shfl_sync(0xffffffffu, extra, 11);
    const int ncls = __shfl_sync(0xffffffffu, extra, 12);
    const int rslot = __shfl_sync(0xffffffffu, extra, 13);
    const bool shard_alive = !(p.n_shards > 1 && ld_volatile(&p.shard_found[shard]));
    // -- eager reads: a consistent read never changes the state, so if any candidate read is consistent
    //    it is linearized immediately and exclusively (verdict- and witness-preserving: any path from
    //    this config can be re-ordered to start with that read).  Not in Knossos; see DESIGN.md.
    int eager_t = -1;
    if (EAGER && shard_alive) {
        unsigned best_inv = 0xffffffffu;  // earliest-invoked consistent read seen by this lane
        int best_t = -1;
        for (int r = 0; r < cand_rounds; ++r) {
            const int t = r * 32 + lane;
            const int32_t* cell = row + ROW_EXTRA + t * SW;
            const int4 op = __ldg(reinterpret_cast<const int4*>(cell));
            bool rd = op.x >= 0 && (op.x & 0xff) == JTB_F_READ && !((w[1] >> t) & 1ull);
            if (rd) {
                int32_t creg = preg;
                int32_t cbal[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) cbal[i] = pbal[i];
                rd = model_step<MODEL>(op, creg, cbal, cell, neg_ok != 0, w[1]);
            }
            if (rd && (unsigned)op.w < best_inv) { best_inv = (unsigned)op.w; best_t = t; }
        }
        const unsigned mn = __reduce_min_sync(0xffffffffu, best_inv);
        if (mn != 0xffffffffu) {
            const unsigned who = __ballot_sync(0xffffffffu, best_inv == mn);
            eager_t = __shfl_sync(0xffffffffu, best_t, __ffs(who) - 1);
        }
    }
    // -- candidates: ops in the open slots
    for (int r = 0; r < cand_rounds && shard_alive; ++r) {
        const int t = r * 32 + lane;
        const int32_t* cell = row + ROW_EXTRA + t * SW;
        const int4 op = __ldg(reinterpret_cast<const int4*>(cell));
        const bool cand = op.x >= 0 && !((w[1] >> t) & 1ull) && (eager_t < 0 || eager_t == t);
        int32_t creg = preg;
        int32_t cbal[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) cbal[i] = pbal[i];
        bool ok = cand && model_step<MODEL>(op, creg, cbal, cell, neg_ok != 0, w[1]);
        const bool is_front = t == rslot;
        uint64_t cw[KW];
#pragma unroll
        for (int i = 0; i < KW; ++i) cw[i] = w[i];
        int cgj = gj;
        // frontier advance, warp-cooperative, for the child that linearizes the frontier op
        const unsigned front_ok = __ballot_sync(0xffffffffu, ok && is_front);
        if (front_ok) {
            uint64_t m = w[1];
            int adv = 0;
            const int32_t* rw = row;
            int32_t ex = extra;
            for (;;) {
                const int32_t word = __shfl_sync(0xffffffffu, ex, lane >> 2);
                const int sl = (word >> (8 * (lane & 3))) & 0xff;
                const bool setb = sl != 0xff && ((m >> sl) & 1ull);
                const unsigned peers = __match_any_sync(0xffffffffu, sl);
                const bool pass = setb && (peers & ((1u << lane) - 1)) == 0;
                const unsigned pm = __ballot_sync(0xffffffffu, pass);
                const int n = pm == 0xffffffffu ? 32 : __ffs(~pm) - 1;
                const uint64_t clr = (lane < n) ? (1ull << sl) : 0ull;
                const uint32_t clo = __reduce_or_sync(0xffffffffu, (uint32_t)clr);
                const uint32_t chi = __reduce_or_sync(0xffffffffu, (uint32_t)(clr >> 32));
                m &= ~((uint64_t)clo | ((uint64_t)chi << 32));
                adv += n;
                if (n < 32) break;
                rw += (size_t)32 * p.row_words;
                ex = __ldg(rw + (lane & 15));
            }
            if (is_front) { cgj = gj + 1 + adv; cw[1] = m; }
        }
        if (ok && !is_front) cw[1] |= 1ull << t;
        cw[0] = KEY_VALID | ((uint64_t)(uint32_t)cgj << 32) |
                ((MODEL == JTB_MODEL_BANK || MODEL == JTB_MODEL_SET) ? 0ull : (uint64_t)(uint32_t)creg);
        int is_new = 0;
        if (ok) {
            if (cgj >= gj_end) {
                // every :ok op of the shard is linearized -> VALID
                if (atomicExch(&p.shard_found[shard], 1) == 0) {
                    if (atomicSub(&ctrl->n_undecided, 1) == 1) atomicCAS(&ctrl->stop, 0, 1);
                }
            } else {
                int plen;
                const int res = table_insert<KW>(p.table, p.slot_mask, cw, &plen);
                my_probes++;
                my_max_probe = max(my_max_probe, plen);
                if (res < 0) {
                    // table exhausted: pause for growth; the child is queued un-inserted (KEY_RETRY)
                    atomicCAS(&ctrl->cause, 0, JTB_CAUSE_TABLE_FULL);
                    atomicCAS(&ctrl->stop, 0, 2);
                    cw[0] |= KEY_RETRY;
                }
                is_new = res != 0;
                if (is_new && cgj > gj) {
                    // witness bookkeeping: furthest frontier reached in this shard
                    const unsigned long long wc = *(volatile unsigned long long*)&*wit_cache;
                    if ((int)(wc >> 32) != shard || (int)(uint32_t)wc < cgj) {
                        *(volatile unsigned long long*)&*wit_cache =
                            ((unsigned long long)(uint32_t)shard << 32) | (uint32_t)cgj;
                        atomicMax(&p.shard_max_rank[shard], cgj);
                    }
                }
            }
        }
        push(is_new != 0, cw, cbal);
    }
    // -- candidates: next member of each crashed-op class
    for (int r = 0; r < cls_rounds && shard_alive && eager_t < 0; ++r) {
        const int c = r * 32 + lane;
        bool cand = c < ncls;
        struct { int first, n, word, shift_width; } cr = {0, 0, 1, 0};
        int4 cop = make_int4(OP_IMPOSSIBLE, 0, 0, 0);
        if (cand) {
            const int4* q = reinterpret_cast<const int4*>(p.classes + cls_base + c);
            const int4 b = __ldg(q + 1);
            cop = __ldg(q);
            cr.first = b.x; cr.n = b.y; cr.word = b.z; cr.shift_width = b.w;
        }
        const int shift = cr.shift_width & 0xff, width = cr.shift_width >> 8;
        uint64_t cw[KW];
        uint64_t field = 0;
#pragma unroll
        for (int i = 0; i < KW; ++i) { cw[i] = w[i]; if (i == cr.word) field = w[i]; }
        const int count = (int)((field >> shift) & ((1ull << width) - 1));
        cand = cand && count < cr.n;
        if (cand) cand = __ldg(p.cls_inv_pos + cr.first + count) < fr_pos;
        int32_t creg = preg;
        int32_t cbal[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) cbal[i] = pbal[i];
        const bool ok = cand && model_step<MODEL>(cop, creg, cbal, nullptr, neg_ok != 0, w[1]);
#pragma unroll
        for (int i = 1; i < KW; ++i) if (i == cr.word) cw[i] += 1ull << shift;
        cw[0] = KEY_VALID | ((uint64_t)(uint32_t)gj << 32) |
                ((MODEL == JTB_MODEL_BANK || MODEL == JTB_MODEL_SET) ? 0ull : (uint64_t)(uint32_t)creg);
        int is_new = 0;
        if (ok) {
            int plen;
            const int res = table_insert<KW>(p.table, p.slot_mask, cw, &plen);
            my_probes++;
            my_max_probe = max(my_max_probe, plen);
            if (res < 0) {
                atomicCAS(&ctrl->cause, 0, JTB_CAUSE_TABLE_FULL);
                atomicCAS(&ctrl->stop, 0, 2);
                cw[0] |= KEY_RETRY;
            }
            is_new = res != 0;
        }
        push(is_new != 0, cw, cbal);
    }
}

// ------------------------------------------------------------------------------------------------
template <int MODEL, int KW>
struct EntryLayout {
    static constexpr bool HAS_BAL = MODEL == JTB_MODEL_BANK;
    static constexpr int EW = KW + (HAS_BAL ? 4 : 0);  // 64-bit words per ring entry
};

#ifndef JTB_WARPS
#define JTB_WARPS 8
#endif
#ifndef JTB_CTAS_EXACT
#define JTB_CTAS_EXACT 4   // resident CTAs/SM for the Knossos-exact space (throughput-bound)
#endif
#ifndef JTB_CTAS_EAGER
#define JTB_CTAS_EAGER 3   // resident CTAs/SM for eager-read searches (latency-bound)
#endif
constexpr int WGL_WARPS = JTB_WARPS;
constexpr int WGL_THREADS = WGL_WARPS * 32;
constexpr unsigned WGL_MAX_DONATE = 64;       // per step, when donating to hungry warps
#ifndef JTB_BATCH
#define JTB_BATCH 32
#endif
constexpr unsigned WGL_BATCH = JTB_BATCH;     // deque entries popped per CTA step; warps self-schedule over them

struct CtaShared {
    int stop;
    unsigned top, bot;              // local LIFO deque (monotonic indices, masked on use)
    unsigned pop_top, don_bot;      // snapshots for this step's readers
    unsigned n_batch, n_don;
    unsigned batch_next;            // self-scheduling cursor over the staged batch
    unsigned ticket_mask;           // warps that currently hold a ring ticket
    unsigned assign_mask;           // warps that receive a new ticket this step
    unsigned n_exp, n_new;          // expansions / new children of the running step
    unsigned backoff;
    unsigned long long ticket_base, don_base;
    unsigned long long wit_cache;   // (shard << 32 | furthest rank): filter for the witness atomicMax
    unsigned long long polls;
    int since_flush;
};

__device__ __forceinline__ uint64_t ld_volatile64(const uint64_t* p) { return *(const volatile uint64_t*)p; }

// MINB = resident CTAs per SM the register budget is cut for: 4 (64 regs, 32 warps/SM) for large,
// throughput-bound searches; 3 (up to 80 regs, fewer spills) for small latency-bound ones.
template <int MODEL, int KW, int MINB, bool EAGER>
__global__ void __launch_bounds__(WGL_THREADS, MINB) wgl_search_kernel(const WglParams p, const int neg_ok) {
    using L = EntryLayout<MODEL, KW>;
    constexpr int EW = L::EW;
    extern __shared__ __align__(16) uint64_t s_deque[];  // deque_cap * EW words, then WGL_BATCH * EW staging
    __shared__ CtaShared sh;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    Ctrl* ctrl = p.ctrl;
    const unsigned cap_mask = p.deque_cap - 1;
    const unsigned high = p.deque_cap / 2;   // donate the oldest entries beyond this; overflow goes to the ring
    uint64_t* const s_batch = s_deque + (size_t)p.deque_cap * EW;

    if (tid == 0) {
        sh.stop = 0; sh.top = sh.bot = 0;
        sh.ticket_mask = 0; sh.n_exp = 0; sh.n_new = 0;
        sh.backoff = 32;
        sh.wit_cache = ~0ull;
        sh.polls = 0; sh.since_flush = 0;
        const unsigned long long now = globaltimer();
        atomicCAS(&ctrl->t0, 0ull, now);
    }
    bool has_ticket = false;
    unsigned long long ticket = 0;
    unsigned long long my_configs = 0, my_probes = 0, my_expansions = 0;
    int my_steps = 0, my_max_probe = 0;
    bool exiting = false;
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
            const bool may_donate = stop == 2 || size > high || (h > t && size > WGL_WARPS);
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
            // ---- donation: deque nearly full, other warps hungry (tickets waiting), or pausing ---------
            const unsigned long long hunger = h > t ? h - t : 0;
            const unsigned free_warps = ~sh.ticket_mask & ((1u << WGL_WARPS) - 1);
            unsigned n_don = 0;
            if (stop == 2) n_don = size;  // pause: all live work must be in the ring
            else if (size > high) n_don = size - p.deque_cap / 4;
            else if (hunger && size > WGL_WARPS)
                n_don = (unsigned)min((unsigned long long)min(size - WGL_WARPS, WGL_MAX_DONATE), hunger);
            sh.n_don = n_don;
            sh.don_bot = sh.bot;
            if (n_don) {
                sh.don_base = atomicAdd(&ctrl->tail, (unsigned long long)n_don);
                sh.bot += n_don;
            }
            // ---- this step's batch: the deepest entries; warps self-schedule over it ----------------------
            const unsigned n_batch = stop ? 0 : min(size - n_don, WGL_BATCH);
            sh.n_batch = n_batch;
            sh.batch_next = 0;
            sh.pop_top = sh.top;
            sh.top -= n_batch;
            // fewer entries than warps: the surplus ticketless warps wait on ring tickets
            unsigned need = 0;
            if (!stop && n_batch < WGL_WARPS) {
                unsigned want = WGL_WARPS - n_batch - (unsigned)__popc(sh.ticket_mask);
                unsigned rest = free_warps;
                while ((int)want > 0 && rest) { const unsigned b = rest & (0u - rest); need |= b; rest ^= b; --want; }
            }
            sh.assign_mask = need;
            if (need) {
                sh.ticket_base = atomicAdd(&ctrl->head, (unsigned long long)__popc(need));
                sh.ticket_mask |= need;
            }
        }
        __syncthreads();  // (B)
        if (sh.stop == 1) break;
        exiting = sh.stop == 2;
        // ---- donation copy: oldest local entries -> ring (payload first, word0 = ready flag last) -----
        {
            const unsigned n_don = sh.n_don;
            for (unsigned i = tid; i < n_don; i += WGL_THREADS) {
                uint64_t* dst = p.ring + ((sh.don_base + i) & p.ring_mask) * EW;
                const uint64_t* src = &s_deque[(size_t)((sh.don_bot + i) & cap_mask) * EW];
#pragma unroll
                for (int k = 1; k < EW; ++k) dst[k] = src[k];
                __threadfence();
                *(volatile uint64_t*)dst = src[0];
            }
        }
        // ---- stage the batch (deepest first) so that pushes may reuse the deque space -------------------
        const unsigned n_batch = sh.n_batch;
        for (unsigned i = tid; i < n_batch * EW; i += WGL_THREADS) {
            const unsigned e = i / EW, k = i % EW;
            s_batch[i] = s_deque[(size_t)((sh.pop_top - 1 - e) & cap_mask) * EW + k];
        }
        if ((sh.assign_mask >> warp) & 1u) {
            ticket = sh.ticket_base + __popc(sh.assign_mask & ((1u << warp) - 1));
            has_ticket = true;
        }
        __syncthreads();  // (C) batch staged, donated entries copied: pushes may reuse the space
        if (exiting) break;
        if (tid == 0) {  // prefetch the control words of the NEXT step behind this step's expansions
            pre_stop = ld_volatile(&ctrl->stop);
            pre_head = ld_volatile(&ctrl->head);
            pre_tail = ld_volatile(&ctrl->tail);
        }

        // ---- self-scheduled expansion: next staged entry, else one poll of my ring ticket ---------------
        bool polled = false;
        unsigned n_done = 0;
        uint64_t w[KW];
        int32_t pbal[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (;;) {
            bool have = false;
            unsigned idx = 0;
            if (lane == 0) idx = atomicAdd(&sh.batch_next, 1u);
            idx = __shfl_sync(0xffffffffu, idx, 0);
            if (idx < n_batch) {
                const uint64_t* e = &s_batch[(size_t)idx * EW];
#pragma unroll
                for (int i = 0; i < KW; ++i) w[i] = e[i];
                if constexpr (L::HAS_BAL) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const uint64_t v = e[KW + i];
                        pbal[2 * i] = (int32_t)(uint32_t)v;
                        pbal[2 * i + 1] = (int32_t)(uint32_t)(v >> 32);
                    }
                }
                have = true;
            } else if (has_ticket && !polled) {
                polled = true;
                uint64_t* slot = p.ring + (ticket & p.ring_mask) * EW;
                w[0] = ld_volatile64(slot);   // warp-uniform: all lanes load the same address
                if (w[0] != 0) {
                    __threadfence();  // acquire: payload words were written before word0
#pragma unroll
                    for (int i = 1; i < KW; ++i) w[i] = ldcg64(slot + i);
                    if constexpr (L::HAS_BAL) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const uint64_t v = ldcg64(slot + KW + i);
                            pbal[2 * i] = (int32_t)(uint32_t)v;
                            pbal[2 * i + 1] = (int32_t)(uint32_t)(v >> 32);
                        }
                    }
                    __syncwarp();
                    if (lane == 0) {
                        *(volatile uint64_t*)slot = 0;  // slot consumed
                        atomicAnd(&sh.ticket_mask, ~(1u << warp));
                    }
                    has_ticket = false;
                    have = true;
                } else if (lane == 0 && warp == 0) {
                    sh.polls++;
                }
            }
            if (!have) break;
            ++n_done;
            // ---------------- expand (warp-synchronous) ---------------------------------------------
            int n_new_total = 0, n_new_local = 0;

            auto push_children = [&](bool is_new, const uint64_t (&cw)[KW], const int32_t (&cbal)[8]) {
                const unsigned newm = __ballot_sync(0xffffffffu, is_new);
                if (newm == 0) return;
                const unsigned n = (unsigned)__popc(newm);
                // reserve space on the CTA deque; if it is full, publish straight to the global ring
                unsigned base = 0;
                int to_ring = 0;
                if (lane == 0) {
                    unsigned old = *(volatile unsigned*)&sh.top;
                    for (;;) {
                        if (old + n - sh.bot > p.deque_cap) { to_ring = 1; break; }
                        const unsigned seen = atomicCAS(&sh.top, old, old + n);
                        if (seen == old) { base = old; break; }
                        old = seen;
                    }
                }
                base = __shfl_sync(0xffffffffu, base, 0);
                to_ring = __shfl_sync(0xffffffffu, to_ring, 0);
                const unsigned my = __popc(newm & ((1u << lane) - 1));
                if (!to_ring) {
                    if (is_new) {
                        uint64_t* e = &s_deque[(size_t)((base + my) & cap_mask) * EW];
#pragma unroll
                        for (int i = 0; i < KW; ++i) e[i] = cw[i];
                        if constexpr (L::HAS_BAL) {
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                e[KW + i] = (uint64_t)(uint32_t)cbal[2 * i] | ((uint64_t)(uint32_t)cbal[2 * i + 1] << 32);
                        }
                    }
                    n_new_local += n;
                } else {
                    unsigned long long rbase = 0;
                    if (lane == 0) {
                        atomicAdd(&ctrl->created, (unsigned long long)n);  // counted before it becomes visible
                        __threadfence();
                        rbase = atomicAdd(&ctrl->tail, (unsigned long long)n);
                    }
                    rbase = __shfl_sync(0xffffffffu, rbase, 0);
                    if (is_new) {
                        uint64_t* dst = p.ring + ((rbase + my) & p.ring_mask) * EW;
#pragma unroll
                        for (int i = 1; i < KW; ++i) dst[i] = cw[i];
                        if constexpr (L::HAS_BAL) {
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                dst[KW + i] = (uint64_t)(uint32_t)cbal[2 * i] | ((uint64_t)(uint32_t)cbal[2 * i + 1] << 32);
                        }
                        __threadfence();
                        *(volatile uint64_t*)dst = cw[0];
                    }
                }
                n_new_total += n;
            };
            bool expand = true;
            if (w[0] & KEY_RETRY) {
                // a child that met a full table (rare: only around a table growth).  It was counted as a config
                // when it was queued; insert it now: already present -> un-count and drop, still full -> re-queue.
                w[0] &= ~KEY_RETRY;
                int res = 0;
                if (lane == 0) {
                    int plen;
                    res = table_insert<KW>(p.table, p.slot_mask, w, &plen);
                }
                res = __shfl_sync(0xffffffffu, res, 0);
                if (res <= 0) {
                    expand = false;
                    if (lane == 0) { if (my_configs) --my_configs; else atomicAdd(&ctrl->configs, ~0ull); }   // -1
                    if (res < 0) {
                        if (lane == 0) {
                            atomicCAS(&ctrl->cause, 0, JTB_CAUSE_TABLE_FULL);
                            atomicCAS(&ctrl->stop, 0, 2);
                        }
                        uint64_t rw[KW];
#pragma unroll
                        for (int i = 0; i < KW; ++i) rw[i] = w[i];
                        rw[0] |= KEY_RETRY;
                        push_children(lane == 0, rw, pbal);
                    }
                }
            }
            if (expand)
                expand_config<MODEL, KW, EAGER>(p, ctrl, neg_ok, w, pbal, lane, &sh.wit_cache, my_probes,
                                                my_max_probe, push_children);
            if (lane == 0) {
                if (n_new_local) atomicAdd(&sh.n_new, (unsigned)n_new_local);
                my_expansions++;
                my_configs += n_new_total;
                if (++my_steps >= 32 || my_configs >= 512) {
                    // amortised global tally: budget (max_configs) and table-load guard
                    my_steps = 0;
                    const unsigned long long tot = atomicAdd(&ctrl->configs, my_configs) + my_configs;
                    my_configs = 0;
                    if (tot >= p.max_configs) {
                        atomicCAS(&ctrl->cause, 0, p.budget_cause);
                        atomicCAS(&ctrl->stop, 0, 2);
                    }
                }
            }
        }
        if (lane == 0 && n_done) atomicAdd(&sh.n_exp, n_done);
    }
    // ---- flush statistics -------------------------------------------------------------------------
    for (int o = 16; o > 0; o >>= 1) {
        my_probes += __shfl_xor_sync(0xffffffffu, my_probes, o);
        my_max_probe = max(my_max_probe, __shfl_xor_sync(0xffffffffu, my_max_probe, o));
    }
    if (lane == 0) {
        atomicAdd(&ctrl->configs, my_configs);
        atomicAdd(&ctrl->probes, my_probes);
        atomicAdd(&ctrl->expansions, my_expansions);
        atomicMax(&ctrl->max_probe_len, (unsigned long long)my_max_probe);
    }
    if (tid == 0) atomicAdd(&ctrl->polls, sh.polls);
}

// Pause/resume support: gathers the live entries (non-zero ring slots in [lo, hi)) of a paused search
// into a fresh ring, in ring order per block (order is immaterial for correctness).
template <int EW>
__global__ void ring_compact_kernel(const uint64_t* __restrict__ old_ring, uint64_t old_mask, unsigned long long lo,
                                    unsigned long long hi, uint64_t* __restrict__ new_ring, uint64_t new_mask,
                                    unsigned long long* __restrict__ new_tail) {
    for (unsigned long long i = lo + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < hi;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint64_t* src = old_ring + (i & old_mask) * EW;
        if (src[0] == 0) continue;
        const unsigned long long o = atomicAdd(new_tail, 1ull);
        uint64_t* dst = new_ring + (o & new_mask) * EW;
#pragma unroll
        for (int k = 0; k < EW; ++k) dst[k] = src[k];
    }
}

// Re-inserts every key of a full table into a larger one (table growth without losing work).
template <int KW>
__global__ void table_rehash_kernel(const uint64_t* __restrict__ old_table, uint64_t old_slots, uint64_t* new_table,
                                    uint64_t new_mask, int* lost = nullptr) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < old_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t k[KW];
#pragma unroll
        for (int w = 0; w < KW; ++w) k[w] = old_table[i * KW + w];
        if (k[0] == 0) continue;
        int plen;
        // a 4x larger table at load <= 1/8 cannot run out of probe slots; if it ever did, a visited key would be lost
        // and the search would re-expand it (wrong counts): the host turns the flag into UNKNOWN
        if (table_insert<KW>(new_table, new_mask, k, &plen) < 0 && lost)
            atomicExch(lost, 1);
    }
}

// knossos :configs — gathers every visited key whose frontier rank is `rank` (two passes: count, then collect).
template <int KW>
__global__ void table_collect_kernel(const uint64_t* __restrict__ table, uint64_t n_slots, uint32_t rank,
                                     uint64_t* __restrict__ out, unsigned long long cap,
                                     unsigned long long* __restrict__ counter) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_slots; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t k0 = table[i * KW];
        if (k0 == 0 || (uint32_t)((k0 >> 32) & RANK_MASK) != rank) continue;
        const unsigned long long o = atomicAdd(counter, 1ull);
        if (o < cap) {
#pragma unroll
            for (int w = 0; w < KW; ++w) out[o * KW + w] = w == 0 ? (k0 & ~KEY_LOCK) : table[i * KW + w];
        }
    }
}

}  // namespace jtb
