// jtb_lifted_witness.cuh — K15: the lifted serial witness (K14's repaired witness, then lift steps where its repairs
// stop because a repair recorded no new ban) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K15 lifted serial witness").  The run is K14's, kernel for kernel, until
// a repair of a NO_WITNESS shard records no ban.  K14 stops such a shard (rw_shard); K15 (lw_shard) marks it lifting
// when it has lift steps left, and the lift step runs on every lifting shard at once, one word read per step:
//   - lw_steal, a warp per failing gap (rw_failing's): sw_solve over the free and the chosen transfers, with the gap's
//     own bans ignored unless lifted before, and P^0 (the reads' invocations alone) in place of P^;
//   - rw_take (K14's) over the lift step's thieves: a thief no smaller thief competes with bans the chosen transfers of
//     its loot in their gaps;
//   - lw_lift, a thread per ban in force: a ban (g, t) whose t the kept thief g took, and that was never lifted, is
//     marked LW_LIFTED in place (the marked key sorts after every ban in force, so K14's binary search over the bans
//     in force never sees it, and "lifted once" is a search of the marked suffix);
//   - lw_merge, lw_end: the lift step's thieves replace K14's; a shard that lifted nothing stops, the others count a
//     repair and a lift step; K14's release, loot and rounds then run unchanged.
// lw_budget ends a shard at max_repairs repairs until it has lifted, at max_repairs + max_lifts after.  The decision,
// node counts, rounds, repairs, bans, lifts and commit_read equal the LW_SEARCH CPU test oracle's.
#pragma once
#include "jtb_repaired_witness.cuh"

namespace jtb {

constexpr unsigned long long LW_LIFTED = 1ull << 63;   // a ban's key, marked lifted (gap < 2^31: the bit is free)

struct LwDev {
    const unsigned long long* lifted = nullptr;   // sorted (gap << 32 | transfer) | LW_LIFTED, the pairs lifted once
    int32_t n_lifted = 0;
};

// (gap i, transfer t) was lifted once
__device__ __forceinline__ bool lw_lifted(const LwDev& l, int32_t i, int32_t t) {
    const unsigned long long k = ((unsigned long long)(uint32_t)i << 32 | (uint32_t)t) | LW_LIFTED;
    int32_t a = 0, b = l.n_lifted;
    while (a < b) {
        const int32_t c = (a + b) >> 1;
        if (l.lifted[c] < k) a = c + 1; else b = c;
    }
    return a < l.n_lifted && l.lifted[a] == k;
}

// the lift filter of gap i's gather: cp(t) > P^0 of i's lower read (r.Ph is P^0), and no ban of i that cannot be
// lifted (a pair banned again after its lift)
__device__ __forceinline__ bool lw_keep(const TpDev& p, const SwDev& w, const RwDev& r, const LwDev& l, int32_t s,
                                        int32_t i, int32_t t) {
    return !(i > p.rs_off[s] && w.t_okcomp[t] <= r.Ph[i - 1]) && !(rw_banned(r, i, t) && lw_lifted(l, i, t));
}

// thread per shard after rw_verdict: a shard still repairing stops at max_repairs repairs until it has lifted, at
// max_repairs + max_lifts after; *act counts the shards left
__global__ void lw_budget(int32_t S, uint8_t* sact, const int32_t* reps, const int32_t* slifts, int32_t max_repairs,
                          int32_t max_lifts, int32_t* act) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || !sact[s]) return;
    if (reps[s] < (slifts[s] ? max_repairs + max_lifts : max_repairs)) return;
    sact[s] = 0;
    atomicSub(act, 1);
}

// thread per shard, in place of rw_shard: a NO_WITNESS shard with no new ban and lift steps left lifts (*n_lifting
// counts them); another shard with no new ban stops; the others count a repair
__global__ void lw_shard(int32_t S, uint8_t* sact, const int32_t* fcause, int32_t* nbs, int32_t* reps, int32_t* bans,
                         const int32_t* slifts, int32_t max_lifts, uint8_t* slift, int32_t* n_lifting) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || !sact[s]) return;
    if (nbs[s] == 0) {
        if (fcause[s] == JTB_CAUSE_NO_WITNESS && slifts[s] < max_lifts) {
            slift[s] = 1;
            atomicAdd(n_lifting, 1);
        } else {
            sact[s] = 0;
        }
        return;
    }
    reps[s]++;
    bans[s] += nbs[s];
    nbs[s] = 0;
}

// warp per failing gap of a lifting shard: the lift step's steal, sw_solve over the free and the chosen transfers that
// pass the lift filter
__global__ void __launch_bounds__(RG_WARPS * 32) lw_steal(RgDev d, TpDev p, SwDev w, RwDev r, LwDev l,
                                                           const uint8_t* __restrict__ slift,
                                                           const uint8_t* __restrict__ failing, uint8_t* thief,
                                                           uint8_t* rel) {
    __shared__ RgWarp smem[RG_WARPS];
    const int lane = threadIdx.x & 31;
    RgWarp& G = smem[threadIdx.x >> 5];
    const int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (wi >= d.m || !failing[wi]) return;
    const int32_t i = (int32_t)wi, s = d.shard[d.ord[i]];
    if (!slift[s]) return;
    int64_t nodes = 0;
    int32_t chosen = 0;
    const bool ok = sw_solve(d, p, w, G, lane, i, [&](int32_t t) {
        return (p.flag[t] & TP_WIN) && p.lo[t] <= i && i <= p.hi[t] && r.kowner[t] == RG_NONE &&
               lw_keep(p, w, r, l, s, i, t);
    }, nodes, chosen);
    if (lane != 0) return;
    atomicAdd(&w.cnt[(int64_t)s * SW_COUNTERS + 3], (unsigned long long)nodes);
    p.pn[i] = chosen;
    thief[i] = ok;
    rel[i] = 1;
}

// thread per ban in force: lifted when its gap is a kept thief of the lift step that took its transfer (the smallest
// gap that chose it) and the pair was never lifted; nls and *n_lift count the lifts
__global__ void lw_lift(int32_t n_ban, RgDev d, SwDev w, LwDev l, const uint8_t* slift, const uint8_t* thief,
                        unsigned long long* ban, int32_t* nls, int32_t* n_lift) {
    const int32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_ban) return;
    const unsigned long long k = ban[e];
    const int32_t g = (int32_t)(k >> 32), t = (int32_t)(uint32_t)k, s = d.shard[d.ord[g]];
    if (!slift[s] || !thief[g] || w.cmin[t] != g || lw_lifted(l, g, t)) return;
    ban[e] = k | LW_LIFTED;
    atomicAdd(&nls[s], 1);
    atomicAdd(n_lift, 1);
}

// thread per gap of a lifting shard: the lift step's thieves replace the repair's
__global__ void lw_merge(int32_t m, RgDev d, const uint8_t* slift, uint8_t* lthief, uint8_t* thief) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m || !slift[d.shard[d.ord[i]]]) return;
    thief[i] = lthief[i];
    lthief[i] = 0;
}

// thread per lifting shard: one that lifted nothing stops; the others count a repair, a lift step, its lifts and bans
__global__ void lw_end(int32_t S, uint8_t* sact, uint8_t* slift, int32_t* nbs, int32_t* nls, int32_t* reps,
                       int32_t* bans, int32_t* slifts, int32_t* snl) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || !slift[s]) return;
    slift[s] = 0;
    if (nls[s] == 0) {
        sact[s] = 0;
    } else {
        reps[s]++;
        bans[s] += nbs[s];
        slifts[s]++;
        snl[s] += nls[s];
    }
    nbs[s] = 0;
    nls[s] = 0;
}

// ---- host ---------------------------------------------------------------------------------------------------------
// The repair loop with its lift steps is run_witness in jtb_witness.cuh, which K15 runs with max_lifts > 0.

}  // namespace jtb
