// jtb_repaired_witness.cuh — K14: the repaired serial witness (K13's witness, then repair rounds that ban the
// (transfer, gap) pairs a failure blames, release their gaps and run the witness rounds again) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K14 repaired serial witness").  The first run is K13's, kernel for kernel
// (tp_stage, tp_finals, sw_init, sw_gaps / sw_fix rounds, sw_tgap, the max-scan, sw_rt, sw_sum, sw_after, sw_rt_id).
// A shard it proves stays as it is.  The others (sact) then repair, all shards together, one word read per repair:
//   - rw_verdict, a thread per shard: VALID shards leave sact; the others keep their failure;
//   - NO_WITNESS: rw_failing, a thread per gap, the gaps the failing round did not explain (or every unfixed gap when
//     max_rounds ran out), the shard's gaps back to their fixed state before that round; rw_steal, a warp per failing
//     gap: sw_solve over the free and the chosen transfers (not banned in the gap, cp > P^); rw_take, a thread per
//     gap: a thief no smaller thief competes with bans the chosen transfers of its loot in their gaps;
//   - REAL_TIME: rw_after_min, rw_sm_in and a min-scan over the reversed positions give SM (the smallest
//     completion of what must follow a gap); rw_rt_blame, a thread per transfer, bans the chosen transfers that break
//     real time;
//   - rw_shard, a thread per shard: a shard with no new ban leaves sact; the new-ban word;
//   - the bans sorted (cub radix sort) and searched by rw_banned; rw_release_g / rw_release_t / rw_loot: released
//     gaps unfixed and their choices owned by no gap, thieves fixed with their loot;
//   - the rounds again (rw_gaps: sw_solve with the ban and P^ filter; sw_fix), P^ per round by rw_gmax and the
//     max-scan; then the check kernels of K13 for the shards in sact.
// The decision, the node counts, rounds, repairs, bans and commit_read equal the RW_SEARCH CPU test oracle's.
#pragma once
#include "jtb_serial_witness.cuh"

namespace jtb {

struct RwDev {
    const uint8_t* sact = nullptr;        // [n_shards] the shard is repairing
    const int32_t* kowner = nullptr;      // [n_t] K12's owner, RG_NONE none (the witness's choices are the others)
    const int32_t* Ph = nullptr;          // [m] P^ at each position
    const unsigned long long* ban = nullptr;   // sorted gap << 32 | transfer
    int32_t n_ban = 0;
};

// (gap i, transfer t) is banned
__device__ __forceinline__ bool rw_banned(const RwDev& r, int32_t i, int32_t t) {
    const unsigned long long k = (unsigned long long)(uint32_t)i << 32 | (uint32_t)t;
    int32_t a = 0, b = r.n_ban;
    while (a < b) {
        const int32_t c = (a + b) >> 1;
        if (r.ban[c] < k) a = c + 1; else b = c;
    }
    return a < r.n_ban && r.ban[a] == k;
}

// the repair filter of gap i's gather: not banned in i, and cp(t) > P^ of i's lower read
__device__ __forceinline__ bool rw_keep(const TpDev& p, const SwDev& w, const RwDev& r, int32_t s, int32_t i,
                                        int32_t t) {
    return !(i > p.rs_off[s] && w.t_okcomp[t] <= r.Ph[i - 1]) && !rw_banned(r, i, t);
}

// warp per unfixed gap: sw_gaps with the repair filter
__global__ void __launch_bounds__(RG_WARPS * 32) rw_gaps(RgDev d, TpDev p, SwDev w, RwDev r) {
    __shared__ RgWarp smem[RG_WARPS];
    const int lane = threadIdx.x & 31;
    RgWarp& G = smem[threadIdx.x >> 5];
    const int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (wi >= d.m || w.fixed[wi]) return;
    const int32_t i = (int32_t)wi, s = d.shard[d.ord[i]];
    int64_t nodes = 0;
    int32_t chosen = 0;
    const bool ok = sw_solve(d, p, w, G, lane, i, [&](int32_t t) {
        return (p.flag[t] & TP_WIN) && p.lo[t] <= i && i <= p.hi[t] && p.owner[t] == RG_NONE && rw_keep(p, w, r, s, i, t);
    }, nodes, chosen);
    if (lane != 0) return;
    atomicAdd(&w.cnt[(int64_t)s * SW_COUNTERS + 3], (unsigned long long)nodes);
    atomicMax(&p.srounds[s], w.round + 1);
    p.pn[i] = chosen;
    if (!ok) atomicMin(&w.sfail[s], i);
}

// thread per transfer: the largest invocation of every gap's owned transfers (P^'s input)
__global__ void rw_gmax(TpDev p, RwDev r, int32_t* __restrict__ gmax) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t || !r.sact[p.t_shard[t]] || p.owner[t] == RG_NONE) return;
    atomicMax(&gmax[p.owner[t]], p.t_inv[t]);
}

// thread per shard: after a run, VALID shards leave sact (and count as valid); the others keep their failure
// (fcause; fkey: the failing gap or K13's real-time key; fid: K13's id key).  The shards still repairing into *act
__global__ void rw_verdict(int32_t S, SwDev w, uint8_t* sact, uint8_t* svalid, int32_t* fcause,
                           unsigned long long* fkey, unsigned long long* fid, int32_t* stot, const int32_t* srounds,
                           int32_t* act) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || !sact[s]) return;
    stot[s] += srounds[s];
    const int32_t f = w.sfail[s] != RG_NONE ? w.sfail[s] : w.sunf[s];
    if (f != RG_NONE) {
        fcause[s] = JTB_CAUSE_NO_WITNESS;
        fkey[s] = (unsigned long long)f;
    } else if (w.rtkey[s] != ~0ull) {
        fcause[s] = JTB_CAUSE_REAL_TIME;
        fkey[s] = w.rtkey[s];
        fid[s] = w.rtid[s];
    } else {
        fcause[s] = 0;
        sact[s] = 0;
        svalid[s] = 1;
        return;
    }
    atomicAdd(act, 1);
}

// thread per gap of a repairing NO_WITNESS shard: the failing gaps, and the gaps back to their state before the failing
// round (sw_fix fixed every gap of the shard); fprev: fixed as the shard's last round started
__global__ void rw_failing(int32_t m, RgDev d, TpDev p, SwDev w, const uint8_t* sact, const int32_t* fcause,
                           const uint8_t* fprev, uint8_t* failing) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    const int32_t s = d.shard[d.ord[i]];
    failing[i] = 0;
    if (!sact[s] || fcause[s] != JTB_CAUSE_NO_WITNESS) return;
    if (w.sfail[s] != RG_NONE) {
        w.fixed[i] = fprev[i];
        failing[i] = !fprev[i] && p.pn[i] == 0;
    } else {
        failing[i] = !w.fixed[i];
    }
}

// warp per failing gap: the steal, sw_solve over the free and the chosen transfers that pass the repair filter
__global__ void __launch_bounds__(RG_WARPS * 32) rw_steal(RgDev d, TpDev p, SwDev w, RwDev r,
                                                           const uint8_t* __restrict__ failing, uint8_t* thief,
                                                           uint8_t* rel) {
    __shared__ RgWarp smem[RG_WARPS];
    const int lane = threadIdx.x & 31;
    RgWarp& G = smem[threadIdx.x >> 5];
    const int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (wi >= d.m || !failing[wi]) return;
    const int32_t i = (int32_t)wi, s = d.shard[d.ord[i]];
    int64_t nodes = 0;
    int32_t chosen = 0;
    const bool ok = sw_solve(d, p, w, G, lane, i, [&](int32_t t) {
        return (p.flag[t] & TP_WIN) && p.lo[t] <= i && i <= p.hi[t] && r.kowner[t] == RG_NONE && rw_keep(p, w, r, s, i, t);
    }, nodes, chosen);
    if (lane != 0) return;
    atomicAdd(&w.cnt[(int64_t)s * SW_COUNTERS + 3], (unsigned long long)nodes);
    p.pn[i] = chosen;
    thief[i] = ok;
    rel[i] = 1;
}

// append the ban (gap g, transfer t) and release g
__device__ __forceinline__ void rw_ban(int32_t g, int32_t t, int32_t s, unsigned long long* ban, int32_t* n_ban,
                                       int32_t* nbs, uint8_t* rel) {
    ban[atomicAdd(n_ban, 1)] = (unsigned long long)(uint32_t)g << 32 | (uint32_t)t;
    atomicAdd(&nbs[s], 1);
    rel[g] = 1;
}

// thread per gap: a thief keeps its loot when no smaller thief took one of it; the chosen transfers of the loot are
// banned in their gaps
__global__ void rw_take(int32_t m, RgDev d, TpDev p, SwDev w, RwDev r, uint8_t* thief, unsigned long long* ban,
                        int32_t* n_ban, int32_t* nbs, uint8_t* rel) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m || !thief[i]) return;
    const int32_t n = p.pn[i], s = d.shard[d.ord[i]];
    const int32_t* ps = p.poss + i * JTB_TP_MAX_GATHER;
    bool keep = true;
    for (int32_t c = 0; c < n && keep; ++c) keep = w.cmin[ps[c]] == i;
    thief[i] = keep;
    if (!keep) return;
    for (int32_t c = 0; c < n; ++c) {
        const int32_t t = ps[c];
        if (p.owner[t] != RG_NONE && r.kowner[t] == RG_NONE) rw_ban(p.owner[t], t, s, ban, n_ban, nbs, rel);
    }
}

// thread per transfer of a repairing REAL_TIME shard: the smallest completion of the :ok transfers after the last read
// that fail
__global__ void rw_after_min(TpDev p, SwDev w, RwDev r, const int32_t* fcause, int32_t* after) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t];
    if (!r.sact[s] || fcause[s] != JTB_CAUSE_REAL_TIME || p.owner[t] != RG_NONE || p.t_fate[t] != JTB_T_OK ||
        !(p.flag[t] & TP_WIN) || w.t_okcomp[t] > w.P[p.rs_off[s + 1] - 1])
        return;
    atomicMin(&after[s], w.t_okcomp[t]);
}

// thread per position: the reversed input of SM, min(cp(r_i), the smallest :ok completion of D_{i+1} or, at the
// shard's last read, of the failing transfers after it)
__global__ void rw_sm_in(RgDev d, TpDev p, SwDev w, const int32_t* after, int32_t* rkey, int32_t* ry) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.m) return;
    const int32_t u = d.ord[i], s = d.shard[u];
    const int32_t next = i + 1 < p.rs_off[s + 1] ? w.gmin[i + 1] : after[s];
    rkey[d.m - 1 - i] = s;
    ry[d.m - 1 - i] = min(d.comp[u], next);
}

// thread per chosen transfer of a repairing REAL_TIME shard: banned in its gap g when it completes by P_g or is invoked
// at or after SM[g]
__global__ void rw_rt_blame(RgDev d, TpDev p, SwDev w, RwDev r, const int32_t* fcause, const int32_t* rsm,
                            unsigned long long* ban, int32_t* n_ban, int32_t* nbs, uint8_t* rel) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t], g = p.owner[t];
    if (!r.sact[s] || fcause[s] != JTB_CAUSE_REAL_TIME || g == RG_NONE || r.kowner[t] != RG_NONE) return;
    const bool early = g > p.rs_off[s] && w.t_okcomp[t] <= w.P[g - 1];
    if (early || p.t_inv[t] >= rsm[d.m - 1 - g]) rw_ban(g, (int32_t)t, s, ban, n_ban, nbs, rel);
}

// thread per shard: a repairing shard with no new ban stops; the others count a repair
__global__ void rw_shard(int32_t S, uint8_t* sact, int32_t* nbs, int32_t* reps, int32_t* bans) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || !sact[s]) return;
    if (nbs[s] == 0) { sact[s] = 0; return; }
    reps[s]++;
    bans[s] += nbs[s];
    nbs[s] = 0;
}

// thread per gap: released gaps of a repairing shard are unfixed; the gaps of the other shards are all fixed
__global__ void rw_release_g(int32_t m, RgDev d, SwDev w, const uint8_t* sact, const uint8_t* rel) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    if (!sact[d.shard[d.ord[i]]]) w.fixed[i] = 1;
    else if (rel[i]) w.fixed[i] = 0;
}

// thread per transfer: a choice of a released gap is owned by no gap
__global__ void rw_release_t(TpDev p, RwDev r, const uint8_t* rel) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t || !r.sact[p.t_shard[t]]) return;
    const int32_t g = p.owner[t];
    if (g != RG_NONE && r.kowner[t] == RG_NONE && rel[g]) p.owner[t] = RG_NONE;
}

// thread per gap: a thief is fixed and owns its loot; the flags are cleared for the next repair
__global__ void rw_loot(int32_t m, RgDev d, TpDev p, SwDev w, const uint8_t* sact, uint8_t* thief, uint8_t* rel) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m) return;
    if (thief[i] && sact[d.shard[d.ord[i]]]) {
        const int32_t* ps = p.poss + i * JTB_TP_MAX_GATHER;
        for (int32_t c = 0; c < p.pn[i]; ++c) p.owner[ps[c]] = (int32_t)i;
        w.fixed[i] = 1;
    }
    thief[i] = 0;
    rel[i] = 0;
}

// thread per shard of sact: a new run's failures cleared, and its committed counts
__global__ void rw_reset(int32_t S, SwDev w, const uint8_t* sact) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S || !sact[s]) return;
    w.sfail[s] = RG_NONE;
    w.sunf[s] = RG_NONE;
    for (int k = 0; k < 3; ++k) w.cnt[(int64_t)s * SW_COUNTERS + k] = 0;
}

// thread per gap, before a round: fixed as the round starts, for the shards no round has failed yet
__global__ void rw_snap(int32_t m, RgDev d, SwDev w, uint8_t* fprev) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < m && w.sfail[d.shard[d.ord[i]]] == RG_NONE) fprev[i] = w.fixed[i];
}

// thread per gap: the unfixed gaps into one word
__global__ void rw_count(int32_t m, SwDev w) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < m && !w.fixed[i]) atomicAdd(w.unfixed, 1);
}

// ---- host ---------------------------------------------------------------------------------------------------------
// The repair loop on the host is run_witness in jtb_witness.cuh, which K14 runs with no lift steps.

}  // namespace jtb
