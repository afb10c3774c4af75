// jtb_level.cuh — the LEVEL engine: the Wing–Gong/Lowe configuration search as a level-synchronous sweep.
//
// Replaces the hot loop of knossos.wgl/analysis (SURVEY.md A.5: `step` over every call entry that may be linearized
// next, then `cache.add((linearized BitSet, model))`) for exhaustive searches.  Same configurations, same keys, same
// per-thread expansion core (jtb_expand.h) as the work-list engine (jtb_wgl.cuh); what differs is the
// ORDER, and what that order buys on an H100:
//
//   depth(config) = number of linearized ops = frontier rank + popcount(open-slot mask) + crashed-class counts is a
//   function of the key, and every move adds exactly one.  So two equal configurations always meet IN THE SAME LEVEL:
//   the visited set only has to live for one level.  The engine keeps two level arrays (ping-pong, coalesced) and ONE
//   small hash window sized to the level (16 slots per configuration, 6-bit epoch tag in every slot, stale entries are
//   simply overwritten: no clearing, no growth, no re-hash, no pause/resume).  At the bench sizes the window is a few
//   MB — the probe stream runs out of the 50 MB L2 instead of HBM — and memory no longer bounds the search:
//   10^10-configuration spaces fit in 80 GB.
//
//   Inside a level, a warp takes 32 configurations: phase 1, one lane per configuration, finds the candidate ops
//   (bit masks from the frontier row); phase 2 hands EVERY child of the 32 configurations to its own lane (prefix sum
//   + k-th-set-bit select), so all probes of the warp are in flight at once and no lane idles on a configuration with
//   fewer children; new children are compacted in shared memory and appended to the next level 32 at a time
//   (one atomic per 32 entries, fully coalesced stores).
//
//   Levels are separated by one grid barrier (monotone counter in HBM).  Narrow levels (<= narrow_max
//   configurations: the start of every search, eager-read searches) are run by CTA 0 alone with __syncthreads()
//   between them while the other CTAs wait at the barrier.
//
// Verdict / witness / configuration count are those of the work-list engines: the first configuration whose frontier
// passes the shard's last return => VALID; an empty level => INVALID with witness = furthest frontier reached;
// configs = sum of the level sizes (every distinct configuration is inserted exactly once).
#pragma once
#include "jtb_expand.h"
#include "jtb_wgl.cuh"

namespace jtb {

#ifndef JTB_LV_WARPS
#define JTB_LV_WARPS 8
#endif
#ifndef JTB_LV_CTAS
#define JTB_LV_CTAS 3
#endif
constexpr int LV_WARPS = JTB_LV_WARPS;
constexpr int LV_THREADS = LV_WARPS * 32;
constexpr int LV_STAGE = 64;        // staged new entries per warp (ring; flushed 32 at a time)
constexpr int LV_MAX_PROBE = 128;
constexpr int LV_CLS_WORDS = 8;     // beam mode: 64-bit words of the per-configuration class mask (512 crashed-op classes
                                    // per key); the exhaustive sweep keeps one word (64 classes, else the work list runs)
// table slots only: bits 56..61 of word 0 hold the epoch of the insertion (a key's rank must stay below 2^24)
constexpr uint64_t LV_TAG_MASK = 0x3full << 56;
constexpr int64_t LV_MAX_RANKS = 1ll << 24;

constexpr int LV_NSEG = 64;         // output segments of a level array (one append counter each: no hot atomic)
constexpr unsigned LV_F_DECIDED = 1, LV_F_GIVEUP = 2, LV_F_RETRY = 4;   // result flags of an attempt (cause: bits 8..)

struct LvSeg {
    alignas(128) unsigned long long n;   // entries appended to this segment of the next level
};
// Beam mode (histories with crashed ops): of every level only the ~beam_w best configurations per undecided shard are
// expanded — fewest crashed ops consumed first, then furthest frontier (relative to the shard's best in that level).
// A beam can only ever find a linearization (VALID); when it dies the host falls back to an exhaustive engine.
constexpr int LV_BEAM_BINS = 1024;      // 16 crashed-op steps x 64 rank steps
constexpr int LV_BEAM_SHARDS = 16;      // beam mode handles histories of at most this many keys
struct LvBeam {
    unsigned hist[3][LV_BEAM_BINS];     // priority histogram of the configurations appended (set = the attempt's output role)
    int min_crashed[3][LV_BEAM_SHARDS]; // per shard: fewest crashed ops consumed among them
    int max_rank[3][LV_BEAM_SHARDS];    //            furthest frontier among them
};
__host__ __device__ inline int lv_beam_key(int crashed, int min_crashed, int rank, int max_rank) {
    int c = crashed - min_crashed, r = max_rank + 2 - rank;
    c = c < 0 ? 0 : (c > 15 ? 15 : c);
    r = r < 0 ? 0 : (r > 63 ? 63 : r);
    return c * 64 + r;   // smaller = better
}

struct LvState {   // identical in every thread of the grid
    unsigned long long level, attempt, n_in, total;
    int epoch, in_idx, boost, stop, cause;
    int s_in, s_out, s_spare;    // roles of the three counter sets: input counts / this attempt's output / being reset
    int contig;                  // the input is still the launch's contiguous run (not segmented)
    unsigned long long win;      // hash window (slots) of the attempt this state describes = lv_window(n_in, boost)
    int beam_thr, beam_frac;     // beam mode: input configurations with a priority key above beam_thr are dropped (-1: keep
                                 // all); of those AT beam_thr a pseudo-random beam_frac / 1024 are kept
    unsigned long long zeroed;   // table slots known to be initialised
};
struct LvRelease {
    alignas(32) unsigned long long gen;
};
struct LvCtrl {
    alignas(128) LvSeg seg[3][LV_NSEG];      // append counters, three sets in rotation (input / output / spare)
    alignas(128) unsigned flags[3][32];      // result flags of the attempt whose output set is [i] (word 0 used)
    alignas(128) LvState pub;                // state after a run of narrow levels (CTA 0 -> everyone)
    alignas(128) int n_undecided;
    int abort;                               // a grid barrier timed out (internal error)
    alignas(128) unsigned long long probes;
    unsigned long long max_probe_len, max_width, max_window, narrow_levels, retries, t0, t1;
    LvState fin;
    // -DJTB_LV_PROF builds only: cycle sums of CTA 0 / warp 0 per section, and per-CTA busy / wait cycles at barriers
    unsigned long long prof[16];
    unsigned long long prof_cta[1024][2];
    int trace[2048][6];      // beam: per attempt (level, n_out, thr, frac, min crashed, max rank of the output)
    alignas(128) LvRelease arrive[1024];     // grid barrier: one arrival word per CTA, watched by CTA 0 ...
    alignas(128) LvRelease release[1024];    // ... and one release word per CTA, written by CTA 0
};

struct LvParams {
    const int32_t* rows;
    const ClassRec* classes;
    const int32_t* cls_inv_pos;
    uint64_t* table;
    uint64_t table_slots;     // capacity (power of two)
    uint64_t* buf[2];         // level arrays, entries of EW words
    uint32_t* aux[2];         // beam mode: crashed ops consumed, one word per entry of buf[]
    LvBeam* beam;             // beam mode: histogram + per-shard trackers
    uint32_t beam_w;          // beam width per undecided shard (0 = exhaustive sweep)
    uint64_t buf_cap;         // entries per array
    uint64_t seg_cap;         // = buf_cap / LV_NSEG: entries per output segment
    LvCtrl* ctrl;
    int* shard_found;
    int* shard_max_rank;
    int row_words, sum_off, n_shards;
    unsigned long long max_configs;
    unsigned long long time_budget_ns;
    LvState init;              // where to start (level 0, or the level a grown relaunch resumes at)
    uint32_t narrow_max;       // a level of at most this many configurations is run by CTA 0 alone
    uint32_t slots_per_config; // window = pow2ceil(n_in * slots_per_config), at least min_slots
    uint64_t min_slots;
};

template <int KW, int EW, bool BAL, bool BEAM>
struct LvScratch {   // per warp, shared memory
    uint64_t w[32][KW];
    uint64_t todo[32], rd_ok[32];
    uint64_t cls_todo[32][BEAM ? LV_CLS_WORDS : 1];   // crashed-op classes (of the configuration's shard) that yield a child
    int32_t bal[BAL ? 32 : 1][8];
    int32_t hdr[32][6];     // fr_pos, shard, gj_end, cls_base, rslot, ncls
    uint32_t start[36];     // exclusive prefix of the child counts; [32] = total
    uint32_t crashed[BEAM ? 32 : 1];   // beam mode: crashed ops consumed by each configuration of the chunk
    uint32_t stage_aux[BEAM ? LV_STAGE : 1];
    // staged new children: the key, and (bank) the parent's lane and the transfer; the balances are built from the
    // parent's S.bal when the entry is flushed, so every chunk flushes what it staged before the next one's phase 1
    uint32_t stage_mv[BAL ? LV_STAGE : 1];   // owner | d << 5 | c << 8
    int32_t stage_amt[BAL ? LV_STAGE : 1];
    uint64_t stage[LV_STAGE][KW];
};

__device__ __forceinline__ int select64(uint64_t m, int k) {   // position of the k-th (0-based) set bit
    const uint32_t lo = (uint32_t)m;
    const int c = __popc(lo);
    return k < c ? (int)__fns(lo, 0, k + 1) : 32 + (int)__fns((uint32_t)(m >> 32), 0, k - c + 1);
}

__device__ __forceinline__ void lv_load_state(LvState& dst, const LvState* src) {   // through L2, word by word
    static_assert(sizeof(LvState) % 8 == 0, "LvState is copied as 64-bit words");
    uint64_t* d = reinterpret_cast<uint64_t*>(&dst);
    const uint64_t* q = reinterpret_cast<const uint64_t*>(src);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(LvState) / 8); ++i) d[i] = ldcg64(q + i);
}

// Probe + insert into the level window.  1 = inserted (new this level), 0 = already present, -1 = window exhausted.
// A slot is free when it is empty or carries another epoch's tag (dead: every level only ever looks for its own keys).
template <int KW>
__device__ __forceinline__ int lv_insert(uint64_t* table, uint64_t mask, const uint64_t (&k)[KW], uint64_t tag, int* plen) {
    uint64_t idx = hash_key<KW>(k) & mask;
    const uint64_t mine0 = k[0] | tag;
    for (int i = 0; i < LV_MAX_PROBE; ++i) {
        uint64_t* slot = table + idx * KW;
        K128 cur = ldcg128(slot);
        for (int round = 0; round < 2; ++round) {
            const bool free_slot = !(cur.lo >> 63) || (cur.lo & LV_TAG_MASK) != tag;
            if (!free_slot) break;
            const K128 mine{KW == 2 ? mine0 : (mine0 | KEY_LOCK), k[1]};
            const K128 old = cas128(slot, cur, mine);
            if (old.lo == cur.lo && old.hi == cur.hi) {
                if constexpr (KW > 2) {
#pragma unroll
                    for (int x = 2; x < KW; ++x) slot[x] = k[x];
                    __threadfence();
                    *(volatile uint64_t*)slot = mine0;   // unlock
                }
                *plen = i + 1;
                return 1;
            }
            cur = old;   // somebody else took the slot in this epoch: compare with what it wrote
        }
        if constexpr (KW == 2) {
            if ((cur.lo & ~LV_TAG_MASK) == k[0] && cur.hi == k[1]) { *plen = i + 1; return 0; }
        } else {
            if ((cur.lo & ~(LV_TAG_MASK | KEY_LOCK)) == k[0] && cur.hi == k[1]) {
                while (cur.lo & KEY_LOCK) cur.lo = ldcg64(slot);
                __threadfence();
                bool same = true;
#pragma unroll
                for (int x = 2; x < KW; ++x) same &= ldcg64(slot + x) == k[x];
                if (same) { *plen = i + 1; return 0; }
            }
        }
        idx = (idx + 1) & mask;
    }
    *plen = LV_MAX_PROBE;
    return -1;
}

// Grid barrier without atomics.  Every CTA publishes its generation in its own arrival word; the threads of CTA 0 each
// watch a few arrival words, and once all have arrived write one release word per CTA; every other CTA polls only its
// own release word.  `gen` is kept by every thread.  Returns false when the wait exceeds 20 s (900 s for the CTAs that
// sit out a run of narrow levels) — a lost CTA would otherwise hang the device: the kernel then ends with ctrl->abort
// set and the host reports an internal error.
#ifdef JTB_LV_PROF
#define LV_PROF(i, t0) do { if (blockIdx.x == 0 && threadIdx.x == 0) { const long long t_ = clock64(); ctrl->prof[i] += t_ - (t0); (t0) = t_; } } while (0)
#else
#define LV_PROF(i, t0) do { } while (0)
#endif

__device__ __forceinline__ bool lv_grid_barrier(LvCtrl* ctrl, unsigned long long& gen, bool patient) {
    __shared__ int s_ok;
    gen++;
    if (threadIdx.x == 0) s_ok = 1;
    __syncthreads();
#ifdef JTB_LV_PROF
    __shared__ long long s_t_leave;
    long long t_arrive = 0;
    if (threadIdx.x == 0) {
        t_arrive = clock64();
        if (gen > 1) ctrl->prof_cta[blockIdx.x][0] += t_arrive - s_t_leave;
    }
#endif
    const unsigned long long limit = patient ? 900000000000ull : 20000000000ull;
    auto wait_for = [&](const unsigned long long* word) {
        unsigned ns = 20, spins = 0;
        unsigned long long t_wait = 0;
        while (ld_volatile(word) < gen) {
            if (patient) { __nanosleep(ns); if (ns < 400) ns += ns; }
            if ((++spins & 0xfff) == 0) {
                const unsigned long long now = globaltimer();
                if (!t_wait) t_wait = now;
                if (now - t_wait > limit || ld_volatile(&ctrl->abort)) { atomicExch(&ctrl->abort, 1); s_ok = 0; return; }
            }
        }
    };
    if (blockIdx.x == 0) {
        __threadfence();
        for (unsigned i = threadIdx.x + 1; i < gridDim.x; i += blockDim.x) wait_for(&ctrl->arrive[i].gen);
        __syncthreads();
        __threadfence();
        for (unsigned i = threadIdx.x + 1; i < gridDim.x; i += blockDim.x) *(volatile unsigned long long*)&ctrl->release[i].gen = gen;
    } else if (threadIdx.x == 0) {
        __threadfence();
        *(volatile unsigned long long*)&ctrl->arrive[blockIdx.x].gen = gen;
        wait_for(&ctrl->release[blockIdx.x].gen);
        __threadfence();
    }
#ifdef JTB_LV_PROF
    if (threadIdx.x == 0) {
        s_t_leave = clock64();
        ctrl->prof_cta[blockIdx.x][1] += s_t_leave - t_arrive;
    }
#endif
    __syncthreads();
    return s_ok != 0;
}

__host__ __device__ inline uint64_t lv_pow2ceil(uint64_t x) {
#if defined(__CUDA_ARCH__)
    return x <= 1 ? 1ull : 1ull << (64 - __clzll((long long)(x - 1)));
#else
    uint64_t s = 1;
    while (s < x) s <<= 1;
    return s;
#endif
}

__host__ __device__ inline uint64_t lv_window(const LvParams& p, unsigned long long n_in, int boost) {
    uint64_t want = (uint64_t)n_in * p.slots_per_config;
    if (want < p.min_slots) want = p.min_slots;
    uint64_t s = lv_pow2ceil(want);
    for (int b = 0; b < boost && s < p.table_slots; ++b) s <<= 2;
    return s < p.table_slots ? s : p.table_slots;
}

// state transition after an attempt — evaluated identically by every thread that needs it.
// cnt = entries appended (sum over the segments), over = some segment ran past its capacity.
__device__ __forceinline__ void lv_advance(const LvParams& p, LvState& st, unsigned long long cnt, bool over, unsigned flags) {
    st.attempt++;
    st.epoch = (st.epoch + 1) & 63;
    const int o_in = st.s_in, o_out = st.s_out, o_spare = st.s_spare;
    if (flags & LV_F_GIVEUP) { st.stop = 2; st.cause = (int)(flags >> 8); return; }
    if (flags & LV_F_RETRY) {
        if (st.win >= p.table_slots) { st.stop = 2; st.cause = JTB_CAUSE_TABLE_FULL; return; }
        st.boost++;
        st.win = lv_window(p, st.n_in, st.boost);
        st.s_out = o_spare; st.s_spare = o_out;   // same level, same input, larger window, new epoch
        return;
    }
    if (over) { st.stop = 2; st.cause = JTB_CAUSE_TABLE_FULL; return; }
    st.total += cnt;
    if (flags & LV_F_DECIDED) { st.stop = 1; return; }
    if (cnt == 0) { st.stop = 1; return; }                        // exhausted: the undecided shards are INVALID
    if (p.max_configs && st.total >= p.max_configs) { st.stop = 2; st.cause = JTB_CAUSE_BUDGET; return; }
    st.level++;
    st.n_in = cnt;
    st.in_idx ^= 1;
    st.contig = 0;
    st.beam_thr = -1;
    st.win = lv_window(p, st.n_in, st.boost);
    st.s_in = o_out; st.s_out = o_spare; st.s_spare = o_in;
}

// NEGOK: the bank model with negative balances allowed (core.clj:217-219, the reference's default) — a transfer never
// fails, so phase 2 needs neither the balances nor the transfer record to build a child's key.
// BEAM: the beam mode (see LvBeam) — its own instantiation, so the exhaustive sweep pays nothing for it.
template <int MODEL, int KW, bool EAGER, bool NEGOK, bool BEAM>
__global__ void __launch_bounds__(LV_THREADS, JTB_LV_CTAS) level_search_kernel(const LvParams p) {
    constexpr bool neg_ok = NEGOK;
    constexpr int CLS_WORDS = BEAM ? LV_CLS_WORDS : 1;
    using L = EntryLayout<MODEL, KW>;
    constexpr int EW = L::EW;
    constexpr bool BAL = L::HAS_BAL;
    constexpr unsigned FULL = 0xffffffffu;
    using Scratch = LvScratch<KW, EW, BAL, BEAM>;
    extern __shared__ __align__(16) unsigned char lv_smem[];
    __shared__ LvState s_state;
    __shared__ unsigned long long s_seg_start[LV_NSEG + 1];   // exclusive prefix of the input segments' counts
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned lt_mask = (1u << lane) - 1;
    Scratch& S = reinterpret_cast<Scratch*>(lv_smem)[warp];
    LvCtrl* ctrl = p.ctrl;
    ExpandTables T;
    T.rows = p.rows; T.classes = p.classes; T.cls_inv_pos = p.cls_inv_pos; T.row_words = p.row_words; T.sum_off = p.sum_off;

    LvState st = p.init;
    unsigned long long bar_gen = 0;
    unsigned long long my_probes = 0;
    int my_max_probe = 0;
    int wit_shard = -1, wit_rank = -1;   // lane-private filter for the witness atomicMax
    if (blockIdx.x == 0 && tid == 0) ctrl->t0 = globaltimer();
    // the first input of a launch is ONE contiguous run at the start of the array
    if (tid <= LV_NSEG) s_seg_start[tid] = tid == 0 ? 0 : st.n_in;
    __syncthreads();

    // Where the idx-th configuration of the level lives: segment by binary search in the prefix, then the offset.
    auto entry_of = [&](const LvState& a, unsigned long long idx, unsigned long long& eidx) -> const uint64_t* {
        int lo = 0, hi = LV_NSEG;       // largest s with seg_start[s] <= idx
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (s_seg_start[mid] <= idx) lo = mid; else hi = mid;
        }
        // (a launch's first input is one contiguous run: prefix [0, n, n, ...] puts all of it in "segment 0" at offset 0)
        eidx = (unsigned long long)lo * p.seg_cap + (idx - s_seg_start[lo]);
        return p.buf[a.in_idx] + eidx * EW;
    };

    // ---- one level attempt over the chunks [first, first + stride, ...) of the input array -------------------
    // Chunk = G configurations for one warp (G = 1, 2, .. 32: the smallest that gives every participating warp at most
    // one chunk, so a narrow level is spread over all warps and each has few children = few probe rounds).
    auto run_attempt = [&](const LvState& a, unsigned first_chunk, unsigned chunk_stride) {
        // G = smallest power of two >= ceil(n_in / stride), at most 32
        unsigned G = 32, g_log = 5;
        if (a.n_in < 32ull * chunk_stride) {
            const unsigned q = ((unsigned)a.n_in + chunk_stride - 1) / chunk_stride;
            g_log = q <= 1 ? 0 : 32 - __clz(q - 1);
            G = 1u << g_log;
        }
        const unsigned n_chunks = (unsigned)((a.n_in + G - 1) >> g_log);
        if (first_chunk >= n_chunks) return;   // nothing for this warp in this level
        uint64_t* out = p.buf[a.in_idx ^ 1];
        unsigned* res_flags = &ctrl->flags[a.s_out][0];
        const unsigned my_seg = first_chunk % LV_NSEG;
        unsigned long long* my_cnt = &ctrl->seg[a.s_out][my_seg].n;
        uint64_t* my_out = out + (unsigned long long)my_seg * p.seg_cap * EW;
        const uint64_t wmask = a.win - 1;
        const uint64_t tag = (uint64_t)a.epoch << 56;
        unsigned stg_head = 0, stg_tail = 0;   // warp-uniform
        int bt_shard = -1, bt_min = 0x7fffffff, bt_max = -1;   // beam: lane-private filter for the tracker atomics
        auto flush = [&](unsigned n) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(my_cnt, (unsigned long long)n);
            base = __shfl_sync(FULL, base, 0);
            if (base + n <= p.seg_cap) {
                uint64_t* dst = my_out + base * EW;
                for (unsigned x = lane; x < n * EW; x += 32) {
                    const unsigned e = x / EW, k = x - e * EW, r = (stg_head + e) % LV_STAGE;
                    if (k < (unsigned)KW) {
                        dst[x] = S.stage[r][k];
                    } else if constexpr (BAL) {   // balances 2i, 2i+1 of the parent, after the transfer
                        const unsigned mv = S.stage_mv[r], i0 = 2 * (k - KW);
                        const int owner = (int)(mv & 31), d = (int)((mv >> 5) & 7), c = (int)((mv >> 8) & 7);
                        const int32_t amt = S.stage_amt[r];
                        int32_t b0 = S.bal[owner][i0], b1 = S.bal[owner][i0 + 1];
                        if (amt) {
                            if ((int)i0 == d) b0 -= amt;
                            if ((int)i0 + 1 == d) b1 -= amt;
                            if ((int)i0 == c) b0 += amt;
                            if ((int)i0 + 1 == c) b1 += amt;
                        }
                        dst[x] = u64_of(b0, b1);
                    }
                }
                if (BEAM && (unsigned)lane < n)
                    p.aux[a.in_idx ^ 1][(unsigned long long)my_seg * p.seg_cap + base + lane] = S.stage_aux[(stg_head + lane) % LV_STAGE];
            }   // else: the count beyond seg_cap is seen by everyone after the barrier (TABLE_FULL -> the host grows)
            stg_head += n;
            __syncwarp();
        };
#ifdef JTB_LV_PROF
        long long tp = clock64();
        if (blockIdx.x == 0 && threadIdx.x == 0) ctrl->prof[8]++;
#endif
        for (unsigned chunk = first_chunk; chunk < n_chunks; chunk += chunk_stride) {
            // ---------------- phase 1: lane = configuration ------------------------------------------------
            const unsigned long long idx = (unsigned long long)chunk * G + lane;
            const bool have = (unsigned)lane < G && idx < a.n_in;
            uint64_t todo = 0;
            unsigned n_cls_children = 0;
            {
                Expander<MODEL, KW, EAGER> X;
                X.todo = 0; X.rd_ok = 0; X.ncls = 0; X.cls_i = 0;
                X.fr_pos = 0; X.shard = 0; X.gj_end = 0; X.cls_base = 0; X.rslot = 0;
                if (have) {
                    unsigned long long eidx;
                    const uint64_t* e = entry_of(a, idx, eidx);
                    unsigned crashed = 0;
                    if constexpr (BEAM) crashed = __ldcg(p.aux[a.in_idx] + eidx);
#pragma unroll
                    for (int i = 0; i < KW; ++i) X.w[i] = ldcg64(e + i);
                    if constexpr (BAL) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const uint64_t v = ldcg64(e + KW + i);
                            X.bal[2 * i] = (int32_t)(uint32_t)v;
                            X.bal[2 * i + 1] = (int32_t)(uint32_t)(v >> 32);
                        }
                    }
                    const int shard = X.load_header(T);
                    bool alive = !(p.n_shards > 1 && ld_volatile(&p.shard_found[shard]));
                    if constexpr (BEAM) {   // aux = priority key << 16 | crashed ops consumed
                        S.crashed[lane] = crashed & 0xffffu;
                        if (a.beam_thr >= 0) {   // outside the beam: not expanded
                            const int key = (int)(crashed >> 16);
                            alive = alive && (key < a.beam_thr ||
                                              (key == a.beam_thr && (int)((hash_key<KW>(X.w) >> 17) & 1023) < a.beam_frac));
                        }
                    }
                    X.begin(T, alive);
                    todo = X.todo;
#pragma unroll
                    for (int cw = 0; cw < CLS_WORDS; ++cw) S.cls_todo[lane][cw] = 0;
                    if (X.cls_i == 0) {   // not decided, not an exclusive eager read: crashed-op classes are candidates
                        uint64_t cw_bits = 0;
                        for (int ci = 0; ci < X.ncls; ++ci) {
                            const int32_t* q = reinterpret_cast<const int32_t*>(T.classes + X.cls_base + ci);
                            const I4 b = ld_i4(q + 4);
                            const int shift = b.w & 0xff, width = b.w >> 8;
                            uint64_t field = 0;
#pragma unroll
                            for (int i = 1; i < KW; ++i) if (i == b.z) field = X.w[i];
                            const int count = (int)((field >> shift) & ((1ull << width) - 1));
                            if (count < b.y && ld_i32(T.cls_inv_pos + b.x + count) < X.fr_pos) { cw_bits |= 1ull << (ci & 63); ++n_cls_children; }
                            if ((ci & 63) == 63 || ci == X.ncls - 1) { S.cls_todo[lane][ci >> 6] = cw_bits; cw_bits = 0; }
                        }
                    }
#pragma unroll
                    for (int i = 0; i < KW; ++i) S.w[lane][i] = X.w[i];
                    if constexpr (BAL) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) S.bal[lane][i] = X.bal[i];
                    }
                    S.rd_ok[lane] = X.rd_ok;
                    S.hdr[lane][0] = X.fr_pos; S.hdr[lane][1] = X.shard; S.hdr[lane][2] = X.gj_end;
                    S.hdr[lane][3] = X.cls_base; S.hdr[lane][4] = X.rslot; S.hdr[lane][5] = X.ncls;
                }
                S.todo[lane] = todo;
            }
            unsigned c = (unsigned)__popcll(todo) + n_cls_children;
            unsigned incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned v = __shfl_up_sync(FULL, incl, o);
                if (lane >= o) incl += v;
            }
            LV_PROF(0, tp);   // phase 1
            S.start[lane] = incl - c;
            const unsigned total = __shfl_sync(FULL, incl, 31);
            if (lane == 0) S.start[32] = total;
            __syncwarp();
            // ---------------- phase 2: lane = child ------------------------------------------------------------
            for (unsigned g0 = 0; g0 < total; g0 += 32) {
                const unsigned g = g0 + lane;
                const bool act = g < total;
                Child<KW> ch;
                bool is_new = false;
                int owner = 0;
                unsigned child_crashed = 0;
                if (act) {
                    int lo = 0, hi = 32;       // largest o with start[o] <= g
                    while (hi - lo > 1) {
                        const int mid = (lo + hi) >> 1;
                        if (S.start[mid] <= g) lo = mid; else hi = mid;
                    }
                    owner = lo;
                    const int k = (int)(g - S.start[owner]);
                    Expander<MODEL, KW, EAGER> Y;
#pragma unroll
                    for (int i = 0; i < KW; ++i) Y.w[i] = S.w[owner][i];
                    if constexpr (BAL && !NEGOK) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) Y.bal[i] = S.bal[owner][i];
                    }
                    Y.rd_ok = S.rd_ok[owner];
                    Y.gj = (int)((Y.w[0] >> 32) & XRANK_MASK);
                    Y.reg = (int32_t)(uint32_t)Y.w[0];
                    Y.row = T.rows + (size_t)Y.gj * T.row_words;
                    Y.fr_pos = S.hdr[owner][0]; Y.shard = S.hdr[owner][1]; Y.gj_end = S.hdr[owner][2];
                    Y.cls_base = S.hdr[owner][3]; Y.rslot = S.hdr[owner][4]; Y.ncls = S.hdr[owner][5];
                    const uint64_t otodo = S.todo[owner];
                    const int ns = __popcll(otodo);
                    bool ok;
                    int t_slot = 0;
                    if constexpr (BEAM) child_crashed = S.crashed[owner] + (k >= ns ? 1u : 0u);
                    if (k < ns) { t_slot = select64(otodo, k); ok = Y.child_slot(T, t_slot, neg_ok, ch, true); }
                    else {   // (k - ns)-th candidate class: find its word, then the bit
                        int kk = k - ns, cw = 0;
                        for (; cw < CLS_WORDS - 1; ++cw) {
                            const int pc = __popcll(S.cls_todo[owner][cw]);
                            if (kk < pc) break;
                            kk -= pc;
                        }
                        ok = Y.child_class(T, cw * 64 + select64(S.cls_todo[owner][cw], kk), neg_ok, ch);
                    }
                    if (ok) {
                        if (ch.done) {
                            // every :ok op of the shard is linearized -> VALID
                            if (atomicExch(&p.shard_found[Y.shard], 1) == 0) {
                                if (atomicSub(&ctrl->n_undecided, 1) == 1) atomicOr(res_flags, LV_F_DECIDED);
                            }
                        } else {
                            int plen;
                            const int r = lv_insert<KW>(p.table, wmask, ch.w, tag, &plen);
                            my_probes++;
                            my_max_probe = max(my_max_probe, plen);
                            if (r < 0) atomicOr(res_flags, LV_F_RETRY);
                            is_new = r == 1;
                            if constexpr (BAL) {
                                if (is_new && ch.d < 0) Y.load_transfer(t_slot, ch);   // only NEW children need the transfer
                            }
                            if (is_new && ch.cgj > Y.gj && (wit_shard != Y.shard || wit_rank < ch.cgj)) {
                                wit_shard = Y.shard; wit_rank = ch.cgj;   // furthest frontier reached: the witness
                                atomicMax(&p.shard_max_rank[Y.shard], ch.cgj);
                            }
                            if (BEAM && is_new) {
                                // priority of the child RELATIVE TO THE INPUT LEVEL's best of its shard (the output level's
                                // own best is only known when the level is complete), and the trackers of the output level
                                LvBeam* bm = p.beam;
                                const int key = lv_beam_key((int)child_crashed, __ldcg(&bm->min_crashed[a.s_in][Y.shard]), ch.cgj,
                                                            __ldcg(&bm->max_rank[a.s_in][Y.shard]));
                                atomicAdd(&bm->hist[a.s_out][key], 1u);
                                child_crashed = min(child_crashed, 0xffffu) | ((unsigned)key << 16);
                                if (bt_shard != Y.shard) { bt_shard = Y.shard; bt_min = 0x7fffffff; bt_max = -1; }
                                const int cc = (int)(child_crashed & 0xffffu);
                                if (cc < bt_min) { bt_min = cc; atomicMin(&bm->min_crashed[a.s_out][Y.shard], bt_min); }
                                if (ch.cgj > bt_max) { bt_max = ch.cgj; atomicMax(&bm->max_rank[a.s_out][Y.shard], bt_max); }
                            }
                        }
                    }
                }
                // ---- stage the new children; append 32 at a time ----
                const unsigned newm = __ballot_sync(FULL, is_new);
                if (newm) {
                    if (is_new) {
                        const unsigned r = (stg_tail + __popc(newm & lt_mask)) % LV_STAGE;
                        uint64_t* e = S.stage[r];
                        if constexpr (BEAM) S.stage_aux[r] = child_crashed;
#pragma unroll
                        for (int i = 0; i < KW; ++i) e[i] = ch.w[i];
                        if constexpr (BAL) {
                            S.stage_mv[r] = (unsigned)owner | ((unsigned)(ch.d & 7) << 5) | ((unsigned)(ch.c & 7) << 8);
                            S.stage_amt[r] = ch.amt;
                        }
                    }
                    stg_tail += __popc(newm);
                    __syncwarp();
                    if (stg_tail - stg_head >= 32) flush(32);
                }
            }
            // the staged balances are built from this chunk's S.bal: flush before the next chunk overwrites it
            if (BAL && stg_tail != stg_head) flush(stg_tail - stg_head);
            __syncwarp();   // the scratch of this chunk is dead
            LV_PROF(1, tp);   // phase 2
        }
        if (stg_tail != stg_head) flush(stg_tail - stg_head);
        LV_PROF(2, tp);       // final flush
    };

    // After an attempt (and the barrier / __syncthreads behind it): ONE warp of the CTA reads the 64 segment counts and
    // the flag word, builds the prefix the next attempt addresses its input with, and the new state.
    auto collect = [&](LvState& a) {
        if (warp == 0) {
            const unsigned long long c0 = ld_volatile(&ctrl->seg[a.s_out][lane].n);
            const unsigned long long c1 = ld_volatile(&ctrl->seg[a.s_out][lane + 32].n);
            unsigned fl = 0;
            if (lane == 0) fl = *(volatile unsigned*)&ctrl->flags[a.s_out][0];
            const bool over = c0 > p.seg_cap || c1 > p.seg_cap;
            unsigned long long i0 = c0, i1 = c1;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long v0 = __shfl_up_sync(FULL, i0, o), v1 = __shfl_up_sync(FULL, i1, o);
                if (lane >= o) { i0 += v0; i1 += v1; }
            }
            const unsigned long long t0 = __shfl_sync(FULL, i0, 31);
            const unsigned long long t1 = __shfl_sync(FULL, i1, 31);
            const bool any_over = __any_sync(FULL, over);
            LvState nx = a;
            if (lane == 0) lv_advance(p, nx, t0 + t1, any_over, fl);
            // beam mode: more configurations than the beam holds -> the largest priority key that still fits
            int thr = -1, frac = 1024;
            if constexpr (BEAM) {
                const unsigned long long cap = (unsigned long long)p.beam_w * (unsigned)max(1, ld_volatile(&ctrl->n_undecided));
                if (t0 + t1 > cap) {
                    unsigned mine = 0;   // lane owns bins [32 lane, 32 lane + 32)
                    const unsigned* hh = p.beam->hist[a.s_out];
#pragma unroll 8
                    for (int i = 0; i < 32; ++i) mine += *(volatile const unsigned*)&hh[lane * 32 + i];
                    unsigned incl_h = mine;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned v = __shfl_up_sync(FULL, incl_h, o);
                        if (lane >= o) incl_h += v;
                    }
                    // first lane whose inclusive count reaches the cap refines inside its 32 bins
                    const unsigned reach = __ballot_sync(FULL, incl_h >= cap);
                    if (reach) {
                        const int wl = __ffs(reach) - 1;
                        if (lane == wl) {
                            unsigned long long run = incl_h - mine;
                            int b = 0;
                            unsigned in_bin = 1;
                            for (; b < 32; ++b) {
                                in_bin = *(volatile const unsigned*)&hh[lane * 32 + b];
                                if (run + in_bin >= cap) break;
                                run += in_bin;
                            }
                            thr = lane * 32 + min(b, 31);
                            // the boundary bin usually holds far more than what is left of the beam: keep a pseudo-random
                            // share of it (chosen by a hash of the whole key, so related configurations are not kept or
                            // dropped together)
                            frac = (int)min(1024ull, (cap - min(cap, run)) * 1024ull / max(in_bin, 1u) + 1ull);
                        }
                        thr = __shfl_sync(FULL, thr, wl);
                        frac = __shfl_sync(FULL, frac, wl);
                    }
                }
            }
            if (lane == 0 && !nx.stop && !((fl & LV_F_RETRY))) { nx.beam_thr = thr; nx.beam_frac = frac; }
#ifdef JTB_LV_PROF
            if (BEAM && blockIdx.x == 0 && lane == 0 && a.attempt < 2048) {
                int* tr = ctrl->trace[a.attempt];
                tr[0] = (int)a.level; tr[1] = (int)(t0 + t1); tr[2] = thr; tr[3] = frac;
                tr[4] = *(volatile int*)&p.beam->min_crashed[a.s_out][0]; tr[5] = *(volatile int*)&p.beam->max_rank[a.s_out][0];
            }
#endif
            // the prefix belongs to the NEXT input = this output, unless the level is repeated (retry): then the old
            // prefix stays (same input)
            const bool repeated = (__shfl_sync(FULL, fl, 0) & LV_F_RETRY) != 0;
            if (!repeated) {
                s_seg_start[lane + 1] = i0;
                s_seg_start[lane + 33] = t0 + i1;
                if (lane == 0) s_seg_start[0] = 0;
            }
            if (lane == 0) s_state = nx;
        }
        __syncthreads();
        a = s_state;
    };

    // ---- cooperative zero-fill of a grown window (the host cleared [0, zeroed_slots)) ---------------------------
    auto zero_fill = [&](uint64_t from, uint64_t to) {
        ulonglong2* t = reinterpret_cast<ulonglong2*>(p.table);
        const uint64_t n16 = (to - from) * KW / 2, off = from * KW / 2;
        for (uint64_t i = (uint64_t)blockIdx.x * LV_THREADS + tid; i < n16; i += (uint64_t)gridDim.x * LV_THREADS)
            t[off + i] = make_ulonglong2(0, 0);
    };
    auto reset_spare = [&](const LvState& a) {   // by ONE warp, during the attempt: the set nobody reads or writes now
        ctrl->seg[a.s_spare][lane].n = 0;
        ctrl->seg[a.s_spare][lane + 32].n = 0;
        if (lane == 0) ctrl->flags[a.s_spare][0] = 0;
        if constexpr (BEAM) {
            for (int i = lane; i < LV_BEAM_BINS; i += 32) p.beam->hist[a.s_spare][i] = 0;
            if (lane < LV_BEAM_SHARDS) { p.beam->min_crashed[a.s_spare][lane] = 0x7fffffff; p.beam->max_rank[a.s_spare][lane] = -1; }
        }
    };

    for (;;) {
        if (st.stop) break;
        const bool narrow = st.n_in <= p.narrow_max;
        {   // a window larger than what is initialised: clear the new part first (wide attempts only; rare)
            const uint64_t win = st.win;
            if (win > st.zeroed) {
                zero_fill(st.zeroed, win);
                st.zeroed = win;
                if (!lv_grid_barrier(ctrl, bar_gen, false)) break;
            }
        }
        if (!narrow) {
            if (blockIdx.x == 0 && warp == LV_WARPS - 1) {
                reset_spare(st);
                if (lane == 0) {
                    if (p.time_budget_ns && globaltimer() - ctrl->t0 > p.time_budget_ns)
                        atomicOr(&ctrl->flags[st.s_out][0], LV_F_GIVEUP | ((unsigned)JTB_CAUSE_BUDGET << 8));
                    if (st.n_in > ctrl->max_width) ctrl->max_width = st.n_in;
                    if (st.win > ctrl->max_window) ctrl->max_window = st.win;
                }
            }
#ifdef JTB_LV_PROF
            long long tw = clock64();
#endif
            run_attempt(st, (unsigned)warp * gridDim.x + blockIdx.x, (unsigned)gridDim.x * LV_WARPS);
            LV_PROF(3, tw);   // whole attempt, CTA 0 thread 0's view
            if (!lv_grid_barrier(ctrl, bar_gen, false)) break;
            LV_PROF(4, tw);   // barrier
            collect(st);
            LV_PROF(5, tw);   // collect
#ifdef JTB_LV_PROF
            if (blockIdx.x == 0 && threadIdx.x == 0) ctrl->prof[9]++;
#endif
            // wide -> narrow: CTA 0 is about to recycle the counter sets on its own; everyone must have read this one
            if (!st.stop && st.n_in <= p.narrow_max && !lv_grid_barrier(ctrl, bar_gen, false)) break;
        } else {
            if (blockIdx.x == 0) {
                // CTA 0 runs narrow levels on its own until the search widens, stops or ends
                for (;;) {
                    if (warp == LV_WARPS - 1) {
                        reset_spare(st);
                        if (lane == 0) {
                            if (p.time_budget_ns && (st.attempt & 63) == 0 && globaltimer() - ctrl->t0 > p.time_budget_ns)
                                atomicOr(&ctrl->flags[st.s_out][0], LV_F_GIVEUP | ((unsigned)JTB_CAUSE_BUDGET << 8));
                            ctrl->narrow_levels++;
                        }
                    }
                    run_attempt(st, (unsigned)warp, (unsigned)LV_WARPS);
                    __syncthreads();
                    collect(st);
                    if (st.stop || st.n_in > p.narrow_max || st.win > st.zeroed) break;
                }
                if (tid == 0) {
                    ctrl->pub = st;
                    __threadfence();
                }
            }
            if (!lv_grid_barrier(ctrl, bar_gen, blockIdx.x != 0)) break;
            if (blockIdx.x != 0) {
                // the others pick the state up and rebuild the input prefix from the counter set that is now the input
                if (tid == 0) lv_load_state(s_state, &ctrl->pub);
                __syncthreads();
                st = s_state;
                if (warp == 0) {
                    const unsigned long long c0 = ld_volatile(&ctrl->seg[st.s_in][lane].n);
                    const unsigned long long c1 = ld_volatile(&ctrl->seg[st.s_in][lane + 32].n);
                    unsigned long long i0 = c0, i1 = c1;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const unsigned long long v0 = __shfl_up_sync(FULL, i0, o), v1 = __shfl_up_sync(FULL, i1, o);
                        if (lane >= o) { i0 += v0; i1 += v1; }
                    }
                    const unsigned long long t0 = __shfl_sync(FULL, i0, 31);
                    s_seg_start[lane + 1] = i0;
                    s_seg_start[lane + 33] = t0 + i1;
                    if (lane == 0) s_seg_start[0] = 0;
                }
                __syncthreads();
            }
        }
    }
    // ---- statistics ---------------------------------------------------------------------------------------
    for (int o = 16; o > 0; o >>= 1) {
        my_probes += __shfl_xor_sync(FULL, my_probes, o);
        my_max_probe = max(my_max_probe, __shfl_xor_sync(FULL, my_max_probe, o));
    }
    if (lane == 0) {
        if (my_probes) atomicAdd(&ctrl->probes, my_probes);
        atomicMax(&ctrl->max_probe_len, (unsigned long long)my_max_probe);
    }
    if (blockIdx.x == 0 && tid == 0) { ctrl->fin = st; ctrl->t1 = globaltimer(); }
}

}  // namespace jtb
