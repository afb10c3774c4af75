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

inline int run_repaired_witness(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                                int64_t max_nodes, int32_t max_rounds, int32_t max_repairs, int32_t flags,
                                int32_t* commit_read, jtb_rw_shard* shards, jtb_rw_result* out, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    if (max_rounds <= 0) max_rounds = JTB_TP_DEFAULT_MAX_ROUNDS;
    if (max_repairs <= 0) max_repairs = JTB_RW_DEFAULT_MAX_REPAIRS;
    TpStage g;
    if (int rc = tp_stage(st, ev0, h, max_nodes, max_rounds, flags, g, err)) return rc;
    const int32_t S = g.S, nT = g.nT, m = g.m;
    std::vector<jtb_tp_shard> tp(std::max(S, 1));
    float ms = 0;
    if (int rc = tp_finals(st, ev0, ev1, h, g, tp.data(), ms, err)) return rc;
    const TlHost& T = g.T;
    std::vector<uint8_t> sok(S, 0);
    bool any = false;
    for (int32_t s = 0; s < S; ++s) {
        jtb_rw_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_reads = tp[s].n_reads;
        o.n_transfers = tp[s].n_transfers;
        o.fail_index = -1;
        o.transfer_id = -1;
        if (tp[s].valid != JTB_VALID) {
            o.valid = JTB_UNKNOWN;
            o.cause = tp[s].cause ? tp[s].cause : tp[s].valid == JTB_INVALID ? JTB_CAUSE_ANOMALY : JTB_CAUSE_UNDECIDED;
        }
        any |= (sok[s] = g.dev[s] && o.valid == JTB_VALID);
    }
    std::vector<int32_t> cr_h(nT, JTB_SW_NEVER);
    if (m > 0 && any) {
        CallAllocs& A = g.A;
        RgDev& x = g.x;
        TpDev& p = g.p;
        SwDev w;
        RwDev r;
        w.t_okcomp = g.d.t_okcomp;
        std::vector<int32_t> rd_cidx(m);
        for (int32_t i = 0; i < m; ++i) rd_cidx[i] = h->index[g.H.r_ev[g.d_of[i]]];
        const int32_t* d_cidx;
        int32_t *d_cr, *kowner, *Ph, *gmaxh, *fcause, *stot, *reps, *bans, *nbs, *after, *rkey, *ry, *rsm, *words;
        uint8_t *sact, *svalid, *fprev, *failing, *thief, *rel, *stmp;
        unsigned long long *fkey, *fid;
        JTB_OK(A.put(&w.sok, sok, st)); JTB_OK(A.put(&d_cidx, rd_cidx, st));
        JTB_OK(A.alloc(&sact, S)); JTB_OK(A.alloc(&svalid, S));
        JTB_OK(cudaMemcpyAsync(sact, w.sok, S, cudaMemcpyDeviceToDevice, st));
        JTB_OK(A.alloc(&w.fixed, m)); JTB_OK(A.alloc(&w.cmin, nT)); JTB_OK(A.alloc(&w.sfail, S));
        JTB_OK(A.alloc(&w.sunf, S)); JTB_OK(A.alloc(&w.unfixed, 1)); JTB_OK(A.alloc(&w.cnt, (size_t)S * SW_COUNTERS));
        JTB_OK(A.alloc(&w.gmax, m)); JTB_OK(A.alloc(&w.gmin, m)); JTB_OK(A.alloc(&w.skey, m));
        JTB_OK(A.alloc(&w.x, m)); JTB_OK(A.alloc(&w.P, m)); JTB_OK(A.alloc(&w.rtkey, S)); JTB_OK(A.alloc(&w.rtid, S));
        JTB_OK(A.alloc(&w.bad, 1)); JTB_OK(A.alloc(&d_cr, nT));
        JTB_OK(A.alloc(&kowner, nT)); JTB_OK(A.alloc(&Ph, m)); JTB_OK(A.alloc(&gmaxh, m));
        JTB_OK(A.alloc(&fcause, S)); JTB_OK(A.alloc(&fkey, S)); JTB_OK(A.alloc(&fid, S)); JTB_OK(A.alloc(&stot, S));
        JTB_OK(A.alloc(&reps, S)); JTB_OK(A.alloc(&bans, S)); JTB_OK(A.alloc(&nbs, S)); JTB_OK(A.alloc(&after, S));
        JTB_OK(A.alloc(&rkey, m)); JTB_OK(A.alloc(&ry, m)); JTB_OK(A.alloc(&rsm, m)); JTB_OK(A.alloc(&words, 2));
        JTB_OK(A.alloc(&fprev, m)); JTB_OK(A.alloc(&failing, m)); JTB_OK(A.alloc(&thief, m)); JTB_OK(A.alloc(&rel, m));
        int64_t* kown;
        JTB_OK(A.alloc(&kown, std::max<int64_t>(g.cells, 1)));
        // the bans: [0, n_ban) sorted in ban[0]; a repair appends at n_ban, then the whole list is sorted into ban[1]
        int64_t ban_cap = std::max<int64_t>(2 * (int64_t)nT, 16);
        unsigned long long* ban[2];
        JTB_OK(A.alloc(&ban[0], ban_cap)); JTB_OK(A.alloc(&ban[1], ban_cap));
        size_t stmp_bytes = 0, sort_bytes = 0;
        JTB_OK(cub::DeviceScan::InclusiveScanByKey(nullptr, stmp_bytes, w.skey, w.x, w.P, MaxOp{}, m,
                                                   cuda::std::equal_to<>{}, st));
        JTB_OK(A.alloc(&stmp, stmp_bytes));
        uint8_t* sort_tmp = nullptr;
        auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };
        JTB_OK(cudaMemsetAsync(w.sfail, 0x7f, (size_t)S * 4, st));   // RG_NONE
        JTB_OK(cudaMemsetAsync(w.sunf, 0x7f, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(w.cnt, 0, (size_t)S * SW_COUNTERS * 8, st));
        JTB_OK(cudaMemsetAsync(w.unfixed, 0, 4, st));
        JTB_OK(cudaMemsetAsync(svalid, 0, S, st));
        JTB_OK(cudaMemsetAsync(fcause, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(stot, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(reps, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(bans, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(nbs, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(thief, 0, m, st));
        JTB_OK(cudaMemsetAsync(rel, 0, m, st));
        JTB_OK(cudaMemcpyAsync(kowner, p.owner, (size_t)nT * 4, cudaMemcpyDeviceToDevice, st));
        JTB_OK(cudaMemcpyAsync(kown, g.own, (size_t)g.cells * 8, cudaMemcpyDeviceToDevice, st));
        r.kowner = kowner;
        r.Ph = Ph;
        r.sact = sact;
        sw_init<<<grid(m, 256), 256, 0, st>>>(x, p, w);
        w.sok = sact;   // from here on the kernels see the shards still repairing
        int32_t n_ban = 0;
        int32_t* d_nban = words + 1;
        JTB_OK(cudaMemsetAsync(words, 0, 8, st));
        for (int32_t rep = 0;; ++rep) {
            // the witness rounds
            int32_t unfixed = 0;
            JTB_OK(cudaMemsetAsync(p.srounds, 0, (size_t)S * 4, st));
            if (rep > 0) {
                JTB_OK(cudaMemsetAsync(w.unfixed, 0, 4, st));
                rw_count<<<grid(m, 256), 256, 0, st>>>(m, w);
            }
            JTB_OK(cudaMemcpyAsync(&unfixed, w.unfixed, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            for (int32_t rd = 0; unfixed > 0 && rd < max_rounds; ++rd) {
                JTB_OK(cudaMemsetAsync(w.cmin, 0x7f, (size_t)nT * 4, st));
                JTB_OK(cudaMemsetAsync(w.unfixed, 0, 4, st));
                rw_snap<<<grid(m, 256), 256, 0, st>>>(m, x, w, fprev);
                w.round = rd;
                if (rep == 0) {
                    sw_gaps<<<grid(m, RG_WARPS), RG_WARPS * 32, 0, st>>>(x, p, w);
                } else {
                    // P^ from the reads and the owned transfers
                    JTB_OK(cudaMemsetAsync(gmaxh, 0x80, (size_t)m * 4, st));
                    if (nT > 0) rw_gmax<<<grid(nT, 256), 256, 0, st>>>(p, r, gmaxh);
                    SwDev wh = w;
                    wh.gmax = gmaxh;
                    sw_scan_in<<<grid(m, 256), 256, 0, st>>>(x, wh);
                    size_t tb = stmp_bytes;
                    JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, w.skey, w.x, Ph, MaxOp{}, m,
                                                               cuda::std::equal_to<>{}, st));
                    rw_gaps<<<grid(m, RG_WARPS), RG_WARPS * 32, 0, st>>>(x, p, w, r);
                }
                sw_fix<<<grid(m, 256), 256, 0, st>>>(m, x, p, w);
                JTB_OK(cudaGetLastError());
                JTB_OK(cudaMemcpyAsync(&unfixed, w.unfixed, 4, cudaMemcpyDeviceToHost, st));
                JTB_OK(cudaStreamSynchronize(st));
            }
            if (unfixed > 0) sw_unfixed<<<grid(m, 256), 256, 0, st>>>(m, x, w);
            // real time and the counters
            JTB_OK(cudaMemsetAsync(w.gmax, 0x80, (size_t)m * 4, st));   // INT_MIN
            JTB_OK(cudaMemsetAsync(w.gmin, 0x7f, (size_t)m * 4, st));   // > every position
            JTB_OK(cudaMemsetAsync(w.rtkey, 0xff, (size_t)S * 8, st));
            JTB_OK(cudaMemsetAsync(w.rtid, 0xff, (size_t)S * 8, st));
            JTB_OK(cudaMemsetAsync(w.bad, 0, 4, st));
            JTB_OK(cudaMemsetAsync(g.own, 0, (size_t)g.cells * 8, st));
            if (nT > 0) sw_tgap<<<grid(nT, 256), 256, 0, st>>>(x, p, w);
            sw_scan_in<<<grid(m, 256), 256, 0, st>>>(x, w);
            size_t tb = stmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, w.skey, w.x, w.P, MaxOp{}, m, cuda::std::equal_to<>{},
                                                       st));
            sw_rt<<<grid(m, 256), 256, 0, st>>>(x, p, w);
            sw_sum<<<grid((int64_t)m * 32, 256), 256, 0, st>>>(x, p, w);
            if (nT > 0) {
                sw_after<<<grid(nT, 256), 256, 0, st>>>(x, p, w);
                sw_rt_id<<<grid(nT, 256), 256, 0, st>>>(x, p, w);
            }
            JTB_OK(cudaMemsetAsync(words, 0, 4, st));
            rw_verdict<<<grid(S, 256), 256, 0, st>>>(S, w, sact, svalid, fcause, fkey, fid, stot, p.srounds, words);
            JTB_OK(cudaGetLastError());
            int32_t hw[2] = {0, 0};
            unsigned int bad = 0;
            JTB_OK(cudaMemcpyAsync(hw, words, 8, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaMemcpyAsync(&bad, w.bad, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            if (bad) { err = "the counters of a serial witness do not add up"; return -1; }
            if (hw[0] == 0 || rep >= max_repairs) break;
            // the blame
            if (n_ban + (int64_t)nT > ban_cap) {
                const int64_t cap = std::max<int64_t>(2 * ban_cap, n_ban + (int64_t)nT);
                unsigned long long *b0, *b1;
                JTB_OK(A.alloc(&b0, cap)); JTB_OK(A.alloc(&b1, cap));
                JTB_OK(cudaMemcpyAsync(b0, ban[0], (size_t)n_ban * 8, cudaMemcpyDeviceToDevice, st));
                ban[0] = b0;
                ban[1] = b1;
                ban_cap = cap;
            }
            r.ban = ban[0];
            r.n_ban = n_ban;
            JTB_OK(cudaMemcpyAsync(g.own, kown, (size_t)g.cells * 8, cudaMemcpyDeviceToDevice, st));
            // P^ for the steals
            JTB_OK(cudaMemsetAsync(gmaxh, 0x80, (size_t)m * 4, st));
            if (nT > 0) rw_gmax<<<grid(nT, 256), 256, 0, st>>>(p, r, gmaxh);
            {
                SwDev wh = w;
                wh.gmax = gmaxh;
                sw_scan_in<<<grid(m, 256), 256, 0, st>>>(x, wh);
                size_t tb2 = stmp_bytes;
                JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb2, w.skey, w.x, Ph, MaxOp{}, m,
                                                           cuda::std::equal_to<>{}, st));
            }
            // NO_WITNESS: the steals
            rw_failing<<<grid(m, 256), 256, 0, st>>>(m, x, p, w, sact, fcause, fprev, failing);
            JTB_OK(cudaMemsetAsync(w.cmin, 0x7f, (size_t)nT * 4, st));
            rw_steal<<<grid(m, RG_WARPS), RG_WARPS * 32, 0, st>>>(x, p, w, r, failing, thief, rel);
            rw_take<<<grid(m, 256), 256, 0, st>>>(m, x, p, w, r, thief, ban[0], d_nban, nbs, rel);
            // REAL_TIME: SM by a min-scan over the reversed positions, then the bans
            JTB_OK(cudaMemsetAsync(after, 0x7f, (size_t)S * 4, st));
            if (nT > 0) rw_after_min<<<grid(nT, 256), 256, 0, st>>>(p, w, r, fcause, after);
            rw_sm_in<<<grid(m, 256), 256, 0, st>>>(x, p, w, after, rkey, ry);
            tb = stmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, rkey, ry, rsm, MinOp{}, m, cuda::std::equal_to<>{},
                                                       st));
            if (nT > 0) rw_rt_blame<<<grid(nT, 256), 256, 0, st>>>(x, p, w, r, fcause, rsm, ban[0], d_nban, nbs, rel);
            rw_shard<<<grid(S, 256), 256, 0, st>>>(S, sact, nbs, reps, bans);
            JTB_OK(cudaGetLastError());
            int32_t total = 0;
            JTB_OK(cudaMemcpyAsync(&total, d_nban, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            if (total == n_ban) break;
            n_ban = total;
            size_t need = 0;
            JTB_OK(cub::DeviceRadixSort::SortKeys(nullptr, need, ban[0], ban[1], n_ban, 0, 64, st));
            if (need > sort_bytes) {
                JTB_OK(A.alloc(&sort_tmp, need));
                sort_bytes = need;
            }
            JTB_OK(cub::DeviceRadixSort::SortKeys(sort_tmp, need, ban[0], ban[1], n_ban, 0, 64, st));
            std::swap(ban[0], ban[1]);
            r.ban = ban[0];
            r.n_ban = n_ban;
            // the release, and the thieves take their loot
            rw_release_g<<<grid(m, 256), 256, 0, st>>>(m, x, w, sact, rel);
            if (nT > 0) rw_release_t<<<grid(nT, 256), 256, 0, st>>>(p, r, rel);
            rw_loot<<<grid(m, 256), 256, 0, st>>>(m, x, p, w, sact, thief, rel);
            rw_reset<<<grid(S, 256), 256, 0, st>>>(S, w, sact);
            JTB_OK(cudaGetLastError());
        }
        // commit_read of the proved shards
        w.sok = svalid;
        if (nT > 0) sw_commit<<<grid(nT, 256), 256, 0, st>>>(x, p, w, d_cidx, d_cr);
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<unsigned long long> cnt_h((size_t)S * SW_COUNTERS), fkey_h(S), fid_h(S);
        std::vector<int32_t> fcause_h(S), stot_h(S), reps_h(S), bans_h(S);
        std::vector<uint8_t> svalid_h(S);
        JTB_OK(cudaMemcpyAsync(cnt_h.data(), w.cnt, cnt_h.size() * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fkey_h.data(), fkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fid_h.data(), fid, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fcause_h.data(), fcause, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(stot_h.data(), stot, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(reps_h.data(), reps, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(bans_h.data(), bans, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(svalid_h.data(), svalid, S, cudaMemcpyDeviceToHost, st));
        if (nT > 0) JTB_OK(cudaMemcpyAsync(cr_h.data(), d_cr, (size_t)nT * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        auto index_at = [&](int32_t at) -> int32_t {   // completion :index of the read at a sorted position
            int32_t rr;
            if (cudaMemcpy(&rr, x.ord + at, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return INT_MIN;
            return rd_cidx[rr];
        };
        for (int32_t s = 0; s < S; ++s) {
            if (!sok[s]) continue;
            jtb_rw_shard& o = shards[s];
            const unsigned long long* c = &cnt_h[(size_t)s * SW_COUNTERS];
            o.nodes = (int64_t)c[3];
            o.rounds = stot_h[s];
            o.repairs = reps_h[s];
            o.n_bans = bans_h[s];
            if (svalid_h[s]) {
                o.n_committed = (int64_t)c[0];
                o.n_committed_crashed = (int64_t)c[1];
                o.n_after = (int64_t)c[2];
                continue;
            }
            o.valid = JTB_UNKNOWN;
            o.cause = fcause_h[s];
            if (o.cause == JTB_CAUSE_NO_WITNESS) {
                o.fail_index = index_at((int32_t)fkey_h[s]);
            } else {
                const int32_t at = (int32_t)(fkey_h[s] >> 1);
                if (fkey_h[s] & 1) {
                    o.fail_index = index_at(at);
                } else {
                    o.transfer_id = (int64_t)(fid_h[s] ^ 0x8000000000000000ull);
                    int32_t t = T.t_off[s];
                    while (T.t_id[t] != o.transfer_id) ++t;
                    o.fail_index = T.t_cidx[t];
                }
            }
            if (o.fail_index == INT_MIN) { err = "cudaMemcpy of a failing read failed"; return -1; }
        }
    }
    // commit_read: the shards with no reads commit their :ok transfers freely; a shard that is not VALID commits none
    for (int32_t s = 0; s < S; ++s) {
        const bool free_ = shards[s].valid == JTB_VALID && g.H.n_reads[s] == 0;
        if (shards[s].valid == JTB_VALID && !free_) continue;
        for (int32_t t = T.t_off[s]; t < T.t_off[s + 1]; ++t)
            cr_h[t] = free_ && T.t_fate[t] == JTB_T_OK ? JTB_SW_FREE : JTB_SW_NEVER;
    }
    if (commit_read && nT > 0) memcpy(commit_read, cr_h.data(), (size_t)nT * 4);
    memset(out, 0, sizeof *out);
    for (int32_t s = 0; s < S; ++s) {
        const jtb_rw_shard& o = shards[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_committed += o.n_committed;
        out->n_committed_crashed += o.n_committed_crashed;
        out->n_after += o.n_after;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
        out->repairs = std::max(out->repairs, (int64_t)o.repairs);
        out->n_bans += o.n_bans;
    }
    roll_up(out, shards, S, ms, t0);
    return 0;
}

}  // namespace jtb
