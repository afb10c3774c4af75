// jtb_lifted_witness.cuh — K15: the lifted serial witness (K14's repaired witness, then lift steps where its repairs
// stop because a repair recorded no new ban) on the device; and the host repair loop K14 and K15 share.
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

inline void lw_set_lifts(jtb_rw_shard&, int32_t, int32_t) {}
inline void lw_set_lifts(jtb_lw_shard& o, int32_t lifts, int32_t n_lifted) {
    o.lifts = lifts;
    o.n_lifted = n_lifted;
}
inline void lw_roll(jtb_rw_result*, const jtb_rw_shard&) {}
inline void lw_roll(jtb_lw_result* out, const jtb_lw_shard& o) {
    out->lifts = std::max(out->lifts, (int64_t)o.lifts);
    out->n_lifted += o.n_lifted;
}
inline void lw_set_lifts(jtb_cw_shard& o, int32_t lifts, int32_t n_lifted) {
    o.lifts = lifts;
    o.n_lifted = n_lifted;
}
inline void lw_roll(jtb_cw_result* out, const jtb_cw_shard& o) {   // K16's class-pass fields too
    out->lifts = std::max(out->lifts, (int64_t)o.lifts);
    out->n_lifted += o.n_lifted;
    out->class_rounds = std::max(out->class_rounds, (int64_t)o.class_rounds);
    out->n_handed += o.n_handed;
}

// what runs after the repairs: nothing for K14 and K15; K16's class pass (jtb_class_witness.cuh), which snapshots
// K12's owners before the witness (pre) and runs on the shards the repairs leave unproved (post)
struct LwNoPass {
    int pre(cudaStream_t, TpStage&, std::string&) { return 0; }
    template <class O>
    int post(cudaStream_t, cudaEvent_t, cudaEvent_t, const jtb_history*, TpStage&, int32_t, O*, std::vector<int32_t>&,
             float&, std::string&) {
        return 0;
    }
};

// K14 (O, R = jtb_rw_shard, jtb_rw_result; max_lifts 0: no lift steps), K15 (jtb_lw_*; max_lifts > 0) and K16
// (jtb_cw_*, with its class pass as Pass)
template <class O, class R, class Pass = LwNoPass>
inline int run_repairs(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, int64_t max_nodes,
                       int32_t max_rounds, int32_t max_repairs, int32_t max_lifts, int32_t* commit_read, O* shards,
                       R* out, int32_t flags, std::string& err, Pass pass = {}) {
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
    if (m > 0)
        if (int rc = pass.pre(st, g, err)) return rc;
    const TlHost& T = g.T;
    std::vector<uint8_t> sok(S, 0);
    bool any = false;
    for (int32_t s = 0; s < S; ++s) {
        O& o = shards[s];
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
        JTB_OK(A.alloc(&rkey, m)); JTB_OK(A.alloc(&ry, m)); JTB_OK(A.alloc(&rsm, m)); JTB_OK(A.alloc(&words, 4));
        JTB_OK(A.alloc(&fprev, m)); JTB_OK(A.alloc(&failing, m)); JTB_OK(A.alloc(&thief, m)); JTB_OK(A.alloc(&rel, m));
        // K15: per shard the lift steps, the pairs lifted, the pairs this step lifts and whether it lifts; per gap the
        // lift step's thieves; P^0
        int32_t *slifts = nullptr, *snl = nullptr, *nls = nullptr, *P0 = nullptr;
        uint8_t *slift = nullptr, *lthief = nullptr;
        if (max_lifts > 0) {
            JTB_OK(A.alloc(&slifts, S)); JTB_OK(A.alloc(&snl, S)); JTB_OK(A.alloc(&nls, S)); JTB_OK(A.alloc(&slift, S));
            JTB_OK(A.alloc(&lthief, m)); JTB_OK(A.alloc(&P0, m));
            JTB_OK(cudaMemsetAsync(slifts, 0, (size_t)S * 4, st));
            JTB_OK(cudaMemsetAsync(snl, 0, (size_t)S * 4, st));
            JTB_OK(cudaMemsetAsync(nls, 0, (size_t)S * 4, st));
            JTB_OK(cudaMemsetAsync(slift, 0, S, st));
            JTB_OK(cudaMemsetAsync(lthief, 0, m, st));
        }
        int64_t* kown;
        JTB_OK(A.alloc(&kown, std::max<int64_t>(g.cells, 1)));
        // the bans: [0, n_ban) sorted in ban[0]; a repair appends at n_ban, then the whole list is sorted into ban[1].
        // K15 marks a lifted ban with LW_LIFTED, so the sort puts the n_lifted lifted pairs after the bans in force
        // (which K14's kernels search as the whole list); a lift step appends a second batch of bans
        const int64_t per_step = (max_lifts > 0 ? 2 : 1) * (int64_t)nT;
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
        LwDev l;
        sw_init<<<grid(m, 256), 256, 0, st>>>(x, p, w);
        if (max_lifts > 0) {   // P^0: the scan of the reads' invocations alone
            JTB_OK(cudaMemsetAsync(gmaxh, 0x80, (size_t)m * 4, st));
            SwDev wh = w;
            wh.gmax = gmaxh;
            sw_scan_in<<<grid(m, 256), 256, 0, st>>>(x, wh);
            size_t tb = stmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, w.skey, w.x, P0, MaxOp{}, m, cuda::std::equal_to<>{},
                                                       st));
        }
        w.sok = sact;   // from here on the kernels see the shards still repairing
        int32_t n_ban = 0, n_lifted = 0;   // bans recorded, and of them lifted
        int32_t* d_nban = words + 1;
        JTB_OK(cudaMemsetAsync(words, 0, 16, st));
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
            if (max_lifts > 0)
                lw_budget<<<grid(S, 256), 256, 0, st>>>(S, sact, reps, slifts, max_repairs, max_lifts, words);
            JTB_OK(cudaGetLastError());
            int32_t hw[2] = {0, 0};
            unsigned int bad = 0;
            JTB_OK(cudaMemcpyAsync(hw, words, 8, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaMemcpyAsync(&bad, w.bad, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            if (bad) { err = "the counters of a serial witness do not add up"; return -1; }
            if (hw[0] == 0 || rep >= max_repairs + max_lifts) break;
            // the blame
            if (n_ban + per_step > ban_cap) {
                const int64_t cap = std::max<int64_t>(2 * ban_cap, n_ban + per_step);
                unsigned long long *b0, *b1;
                JTB_OK(A.alloc(&b0, cap)); JTB_OK(A.alloc(&b1, cap));
                JTB_OK(cudaMemcpyAsync(b0, ban[0], (size_t)n_ban * 8, cudaMemcpyDeviceToDevice, st));
                ban[0] = b0;
                ban[1] = b1;
                ban_cap = cap;
            }
            r.ban = ban[0];
            r.n_ban = n_ban - n_lifted;
            l.lifted = ban[0] + r.n_ban;
            l.n_lifted = n_lifted;
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
            if (max_lifts > 0) {
                JTB_OK(cudaMemsetAsync(words + 2, 0, 8, st));
                lw_shard<<<grid(S, 256), 256, 0, st>>>(S, sact, fcause, nbs, reps, bans, slifts, max_lifts, slift,
                                                       words + 2);
            } else {
                rw_shard<<<grid(S, 256), 256, 0, st>>>(S, sact, nbs, reps, bans);
            }
            JTB_OK(cudaGetLastError());
            int32_t bw[3] = {0, 0, 0};   // bans recorded, shards lifting, bans lifted
            JTB_OK(cudaMemcpyAsync(bw, d_nban, max_lifts > 0 ? 8 : 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            const int32_t total = bw[0];
            if (bw[1] > 0) {
                // the lift step of the shards whose repair recorded no ban: the steals again with the lift filter and
                // P^0; K14's take bans the chosen loot of the kept thieves; then the lifts, a thread per ban in force
                RwDev r0 = r;
                r0.Ph = P0;
                JTB_OK(cudaMemsetAsync(w.cmin, 0x7f, (size_t)nT * 4, st));
                lw_steal<<<grid(m, RG_WARPS), RG_WARPS * 32, 0, st>>>(x, p, w, r0, l, slift, failing, lthief, rel);
                rw_take<<<grid(m, 256), 256, 0, st>>>(m, x, p, w, r, lthief, ban[0], d_nban, nbs, rel);
                if (r.n_ban > 0)
                    lw_lift<<<grid(r.n_ban, 256), 256, 0, st>>>(r.n_ban, x, w, l, slift, lthief, ban[0], nls, words + 3);
                lw_merge<<<grid(m, 256), 256, 0, st>>>(m, x, slift, lthief, thief);
                lw_end<<<grid(S, 256), 256, 0, st>>>(S, sact, slift, nbs, nls, reps, bans, slifts, snl);
                JTB_OK(cudaGetLastError());
                JTB_OK(cudaMemcpyAsync(bw, d_nban, 12, cudaMemcpyDeviceToHost, st));
                JTB_OK(cudaStreamSynchronize(st));
            }
            if (total == n_ban && bw[2] == 0) break;
            n_ban = bw[0];
            n_lifted += bw[2];
            size_t need = 0;
            JTB_OK(cub::DeviceRadixSort::SortKeys(nullptr, need, ban[0], ban[1], n_ban, 0, 64, st));
            if (need > sort_bytes) {
                JTB_OK(A.alloc(&sort_tmp, need));
                sort_bytes = need;
            }
            JTB_OK(cub::DeviceRadixSort::SortKeys(sort_tmp, need, ban[0], ban[1], n_ban, 0, 64, st));
            std::swap(ban[0], ban[1]);
            r.ban = ban[0];
            r.n_ban = n_ban - n_lifted;
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
        std::vector<int32_t> fcause_h(S), stot_h(S), reps_h(S), bans_h(S), lifts_h(S, 0), snl_h(S, 0);
        std::vector<uint8_t> svalid_h(S);
        JTB_OK(cudaMemcpyAsync(cnt_h.data(), w.cnt, cnt_h.size() * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fkey_h.data(), fkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fid_h.data(), fid, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fcause_h.data(), fcause, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(stot_h.data(), stot, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(reps_h.data(), reps, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(bans_h.data(), bans, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(svalid_h.data(), svalid, S, cudaMemcpyDeviceToHost, st));
        if (max_lifts > 0) {
            JTB_OK(cudaMemcpyAsync(lifts_h.data(), slifts, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaMemcpyAsync(snl_h.data(), snl, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        }
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
            O& o = shards[s];
            const unsigned long long* c = &cnt_h[(size_t)s * SW_COUNTERS];
            o.nodes = (int64_t)c[3];
            o.rounds = stot_h[s];
            o.repairs = reps_h[s];
            o.n_bans = bans_h[s];
            lw_set_lifts(o, lifts_h[s], snl_h[s]);
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
    if (m > 0)
        if (int rc = pass.post(st, ev0, ev1, h, g, max_rounds, shards, cr_h, ms, err)) return rc;
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
        const O& o = shards[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_committed += o.n_committed;
        out->n_committed_crashed += o.n_committed_crashed;
        out->n_after += o.n_after;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
        out->repairs = std::max(out->repairs, (int64_t)o.repairs);
        out->n_bans += o.n_bans;
        lw_roll(out, o);
    }
    roll_up(out, shards, S, ms, t0);
    return 0;
}

inline int run_repaired_witness(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                                int64_t max_nodes, int32_t max_rounds, int32_t max_repairs, int32_t flags,
                                int32_t* commit_read, jtb_rw_shard* shards, jtb_rw_result* out, std::string& err) {
    return run_repairs(st, ev0, ev1, h, max_nodes, max_rounds, max_repairs, 0, commit_read, shards, out, flags, err);
}

inline int run_lifted_witness(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                              int64_t max_nodes, int32_t max_rounds, int32_t max_repairs, int32_t max_lifts,
                              int32_t flags, int32_t* commit_read, jtb_lw_shard* shards, jtb_lw_result* out,
                              std::string& err) {
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    return run_repairs(st, ev0, ev1, h, max_nodes, max_rounds, max_repairs, max_lifts, commit_read, shards, out, flags,
                       err);
}

}  // namespace jtb
