// jtb_witness.cuh — the host driver of the witness checks K13–K17 (run_witness).
//
// One driver runs every rung; the five entry points (jtb_check_*_witness in jtb_abi.cu) differ only in their budgets
// and their pass:
//   - K13: no repairs and no lifts, so the loop ends after the first witness (jtb_serial_witness.cuh);
//   - K14: max_repairs repairs (jtb_repaired_witness.cuh);
//   - K15: and max_lifts lift steps (jtb_lifted_witness.cuh);
//   - K16: and CwPass, the class pass on the shards K15 leaves unproved (jtb_class_witness.cuh);
//   - K17: and LkPass, CwPass then the lookup pass (jtb_lookup_witness.cuh).
// The driver: K12's stage and finals (tp_stage, tp_finals); the pass's pre; sw_init; per run the witness rounds (sw_gaps
// in the first run, rw_gaps with P^ after a repair; sw_fix), the real time and re-sum (sw_real_time, sw_rt_id) and
// rw_verdict; between runs, while a shard repairs, the blame, the lift step, the ban sort, the release and the loot;
// then sw_commit of the proved shards, the read-back and the failure decode; the pass's post; commit_read of the
// shards the device does not prove; the roll-up.  It fills one jtb_lk_shard per shard and one jtb_lk_result;
// run_witness_as narrows them to an entry point's ABI structs, which are byte prefixes of K17's (asserted below).
#pragma once
#include <cstddef>
#include <type_traits>

#include "jtb_lookup_witness.cuh"

namespace jtb {

// The narrower witness records are byte prefixes of K17's: every field at K17's offset and of K17's type, each
// shard record ending where K17's next field starts, each result's int64 block where K17's next field starts (the two
// doubles are copied by name).
#define JTB_SW_SHARD(X, T)                                                                                            \
    X(T, valid) X(T, cause) X(T, n_reads) X(T, n_transfers) X(T, n_committed) X(T, n_committed_crashed) X(T, n_after) \
    X(T, nodes) X(T, rounds) X(T, fail_index) X(T, transfer_id)
#define JTB_RW_SHARD(X, T) JTB_SW_SHARD(X, T) X(T, repairs) X(T, n_bans)
#define JTB_LW_SHARD(X, T) JTB_RW_SHARD(X, T) X(T, lifts) X(T, n_lifted)
#define JTB_CW_SHARD(X, T) JTB_LW_SHARD(X, T) X(T, class_cause) X(T, class_rounds) X(T, n_handed)
#define JTB_SW_RESULT(X, T)                                                                                           \
    X(T, valid) X(T, n_failures) X(T, n_reads) X(T, n_transfers) X(T, n_committed) X(T, n_committed_crashed)          \
    X(T, n_after) X(T, nodes) X(T, rounds)
#define JTB_RW_RESULT(X, T) JTB_SW_RESULT(X, T) X(T, repairs) X(T, n_bans)
#define JTB_LW_RESULT(X, T) JTB_RW_RESULT(X, T) X(T, lifts) X(T, n_lifted)
#define JTB_CW_RESULT(X, T) JTB_LW_RESULT(X, T) X(T, class_rounds) X(T, n_handed)
#define JTB_PREFIX(T, W, f)                                                                                           \
    static_assert(offsetof(T, f) == offsetof(W, f) && std::is_same<decltype(T::f), decltype(W::f)>::value,           \
                  #T "::" #f " is not where " #W " has it");
#define JTB_LK_SHARD_PREFIX(T, f) JTB_PREFIX(T, jtb_lk_shard, f)
#define JTB_LK_RESULT_PREFIX(T, f) JTB_PREFIX(T, jtb_lk_result, f)
JTB_SW_SHARD(JTB_LK_SHARD_PREFIX, jtb_sw_shard)
JTB_RW_SHARD(JTB_LK_SHARD_PREFIX, jtb_rw_shard)
JTB_LW_SHARD(JTB_LK_SHARD_PREFIX, jtb_lw_shard)
JTB_CW_SHARD(JTB_LK_SHARD_PREFIX, jtb_cw_shard)
JTB_SW_RESULT(JTB_LK_RESULT_PREFIX, jtb_sw_result)
JTB_RW_RESULT(JTB_LK_RESULT_PREFIX, jtb_rw_result)
JTB_LW_RESULT(JTB_LK_RESULT_PREFIX, jtb_lw_result)
JTB_CW_RESULT(JTB_LK_RESULT_PREFIX, jtb_cw_result)
static_assert(sizeof(jtb_sw_shard) == offsetof(jtb_lk_shard, repairs) &&
                  sizeof(jtb_rw_shard) == offsetof(jtb_lk_shard, lifts) &&
                  sizeof(jtb_lw_shard) == offsetof(jtb_lk_shard, class_cause) &&
                  sizeof(jtb_cw_shard) == offsetof(jtb_lk_shard, lookup_cause) &&
                  offsetof(jtb_sw_result, seconds_kernel) == offsetof(jtb_lk_result, repairs) &&
                  offsetof(jtb_rw_result, seconds_kernel) == offsetof(jtb_lk_result, lifts) &&
                  offsetof(jtb_lw_result, seconds_kernel) == offsetof(jtb_lk_result, class_rounds) &&
                  offsetof(jtb_cw_result, seconds_kernel) == offsetof(jtb_lk_result, n_lookups_placed),
              "a narrower witness record holds more than its prefix of K17's");
#undef JTB_LK_RESULT_PREFIX
#undef JTB_LK_SHARD_PREFIX
#undef JTB_PREFIX
#undef JTB_CW_RESULT
#undef JTB_LW_RESULT
#undef JTB_RW_RESULT
#undef JTB_SW_RESULT
#undef JTB_CW_SHARD
#undef JTB_LW_SHARD
#undef JTB_RW_SHARD
#undef JTB_SW_SHARD

// what runs after the repairs: nothing for K13, K14 and K15
struct NoPass {
    int pre(cudaStream_t, TpStage&, std::string&) { return 0; }
    int post(cudaStream_t, cudaEvent_t, cudaEvent_t, const jtb_history*, TpStage&, int32_t, jtb_lk_shard*,
             std::vector<int32_t>&, float&, std::string&) {
        return 0;
    }
};

// K13–K17 with resolved budgets (0: none; max_repairs + max_lifts = 0 skips the repair state); Pass's pre runs after
// tp_finals on a call with device reads, its post after the read-back of every call
template <class Pass>
inline int run_witness(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, int64_t max_nodes,
                       int32_t max_rounds, int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t* commit_read,
                       jtb_lk_shard* shards, jtb_lk_result* out, Pass& pass, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (max_rounds <= 0) max_rounds = JTB_TP_DEFAULT_MAX_ROUNDS;
    const bool repair = max_repairs + max_lifts > 0;
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
        jtb_lk_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_reads = tp[s].n_reads;
        o.n_transfers = tp[s].n_transfers;
        o.fail_index = o.lookup_fail_index = -1;
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
        if (int rc = sw_alloc(st, g, sok, w, err)) return rc;
        const std::vector<int32_t> rd_cidx = sw_rd_cidx(h, g);
        const int32_t* d_cidx;
        int32_t *d_cr, *fcause, *stot, *reps, *bans, *words;
        uint8_t *sact, *svalid, *stmp;
        unsigned long long *fkey, *fid;
        JTB_OK(A.put(&d_cidx, rd_cidx, st)); JTB_OK(A.alloc(&d_cr, nT));
        JTB_OK(A.alloc(&sact, S)); JTB_OK(A.alloc(&svalid, S));
        JTB_OK(cudaMemcpyAsync(sact, w.sok, S, cudaMemcpyDeviceToDevice, st));
        JTB_OK(A.alloc(&fcause, S)); JTB_OK(A.alloc(&fkey, S)); JTB_OK(A.alloc(&fid, S)); JTB_OK(A.alloc(&stot, S));
        JTB_OK(A.alloc(&reps, S)); JTB_OK(A.alloc(&bans, S)); JTB_OK(A.alloc(&words, 4));
        // K14: K12's owners and owned counters, P^, the failing gaps, thieves and released gaps, the REAL_TIME blame's
        // scan and the bans.  The bans: [0, n_ban) sorted in ban[0]; a repair appends at n_ban, then the whole list is
        // sorted into ban[1].  K15 marks a lifted ban with LW_LIFTED, so the sort puts the n_lifted lifted pairs after
        // the bans in force (which K14's kernels search as the whole list); a lift step appends a second batch of bans
        int32_t *kowner = nullptr, *Ph = nullptr, *gmaxh = nullptr, *nbs = nullptr, *after = nullptr, *rkey = nullptr,
                *ry = nullptr, *rsm = nullptr;
        uint8_t *fprev = nullptr, *failing = nullptr, *thief = nullptr, *rel = nullptr;
        int64_t* kown = nullptr;
        const int64_t per_step = (max_lifts > 0 ? 2 : 1) * (int64_t)nT;
        int64_t ban_cap = std::max<int64_t>(2 * (int64_t)nT, 16);
        unsigned long long* ban[2] = {nullptr, nullptr};
        if (repair) {
            JTB_OK(A.alloc(&kowner, nT)); JTB_OK(A.alloc(&Ph, m)); JTB_OK(A.alloc(&gmaxh, m)); JTB_OK(A.alloc(&nbs, S));
            JTB_OK(A.alloc(&after, S)); JTB_OK(A.alloc(&rkey, m)); JTB_OK(A.alloc(&ry, m)); JTB_OK(A.alloc(&rsm, m));
            JTB_OK(A.alloc(&fprev, m)); JTB_OK(A.alloc(&failing, m)); JTB_OK(A.alloc(&thief, m));
            JTB_OK(A.alloc(&rel, m)); JTB_OK(A.alloc(&kown, std::max<int64_t>(g.cells, 1)));
            JTB_OK(A.alloc(&ban[0], ban_cap)); JTB_OK(A.alloc(&ban[1], ban_cap));
            JTB_OK(cudaMemsetAsync(nbs, 0, (size_t)S * 4, st));
            JTB_OK(cudaMemsetAsync(thief, 0, m, st));
            JTB_OK(cudaMemsetAsync(rel, 0, m, st));
            JTB_OK(cudaMemcpyAsync(kowner, p.owner, (size_t)nT * 4, cudaMemcpyDeviceToDevice, st));
            JTB_OK(cudaMemcpyAsync(kown, g.own, (size_t)g.cells * 8, cudaMemcpyDeviceToDevice, st));
        }
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
        size_t stmp_bytes = 0, sort_bytes = 0;
        JTB_OK(cub::DeviceScan::InclusiveScanByKey(nullptr, stmp_bytes, w.skey, w.x, w.P, MaxOp{}, m,
                                                   cuda::std::equal_to<>{}, st));
        JTB_OK(A.alloc(&stmp, stmp_bytes));
        uint8_t* sort_tmp = nullptr;
        auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };
        JTB_OK(cudaMemsetAsync(svalid, 0, S, st));
        JTB_OK(cudaMemsetAsync(fcause, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(stot, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(reps, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(bans, 0, (size_t)S * 4, st));
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
                if (repair) rw_snap<<<grid(m, 256), 256, 0, st>>>(m, x, w, fprev);
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
            if (int rc = sw_real_time(st, g, w, stmp, stmp_bytes, err)) return rc;
            if (nT > 0) sw_rt_id<<<grid(nT, 256), 256, 0, st>>>(x, p, w);
            JTB_OK(cudaMemsetAsync(words, 0, 4, st));
            rw_verdict<<<grid(S, 256), 256, 0, st>>>(S, w, sact, svalid, fcause, fkey, fid, stot, p.srounds, words);
            if (max_lifts > 0)
                lw_budget<<<grid(S, 256), 256, 0, st>>>(S, sact, reps, slifts, max_repairs, max_lifts, words);
            JTB_OK(cudaGetLastError());
            if (rep >= max_repairs + max_lifts) break;   // the last run's counters are checked with the read-back
            int32_t hw[2] = {0, 0};
            unsigned int bad = 0;
            JTB_OK(cudaMemcpyAsync(hw, words, 8, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaMemcpyAsync(&bad, w.bad, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            if (bad) { err = "the counters of a serial witness do not add up"; return -1; }
            if (hw[0] == 0) break;
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
                size_t tb = stmp_bytes;
                JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, w.skey, w.x, Ph, MaxOp{}, m,
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
            size_t tb = stmp_bytes;
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
        unsigned int bad = 0;
        JTB_OK(cudaMemcpyAsync(cnt_h.data(), w.cnt, cnt_h.size() * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fkey_h.data(), fkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fid_h.data(), fid, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(fcause_h.data(), fcause, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(stot_h.data(), stot, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(reps_h.data(), reps, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(bans_h.data(), bans, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(svalid_h.data(), svalid, S, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(&bad, w.bad, 4, cudaMemcpyDeviceToHost, st));
        if (max_lifts > 0) {
            JTB_OK(cudaMemcpyAsync(lifts_h.data(), slifts, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaMemcpyAsync(snl_h.data(), snl, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        }
        if (nT > 0) JTB_OK(cudaMemcpyAsync(cr_h.data(), d_cr, (size_t)nT * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        if (bad) { err = "the counters of a serial witness do not add up"; return -1; }
        auto index_at = [&](int32_t at) -> int32_t {   // completion :index of the read at a sorted position
            int32_t rr;
            if (cudaMemcpy(&rr, x.ord + at, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return INT_MIN;
            return rd_cidx[rr];
        };
        for (int32_t s = 0; s < S; ++s) {
            if (!sok[s]) continue;
            jtb_lk_shard& o = shards[s];
            const unsigned long long* c = &cnt_h[(size_t)s * SW_COUNTERS];
            o.nodes = (int64_t)c[3];
            o.rounds = stot_h[s];
            o.repairs = reps_h[s];
            o.n_bans = bans_h[s];
            o.lifts = lifts_h[s];
            o.n_lifted = snl_h[s];
            if (svalid_h[s]) {
                o.n_committed = (int64_t)c[0];
                o.n_committed_crashed = (int64_t)c[1];
                o.n_after = (int64_t)c[2];
                continue;
            }
            // the failure: the failing gap (NO_WITNESS), or K13's real-time key, the read at a position or the
            // smallest failing transfer id
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
        const jtb_lk_shard& o = shards[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_committed += o.n_committed;
        out->n_committed_crashed += o.n_committed_crashed;
        out->n_after += o.n_after;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
        out->repairs = std::max(out->repairs, (int64_t)o.repairs);
        out->n_bans += o.n_bans;
        out->lifts = std::max(out->lifts, (int64_t)o.lifts);
        out->n_lifted += o.n_lifted;
        out->class_rounds = std::max(out->class_rounds, (int64_t)o.class_rounds);
        out->n_handed += o.n_handed;
        out->n_lookups_placed += o.n_lookups_placed;
    }
    roll_up(out, shards, S, ms, t0);
    return 0;
}

// run_witness narrowed to an entry point's shard and result structs; the entry point resolves the budgets' defaults
template <class Shard, class Result, class Pass = NoPass>
inline int run_witness_as(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, int64_t max_nodes,
                          int32_t max_rounds, int32_t max_repairs, int32_t max_lifts, int32_t flags,
                          int32_t* commit_read, Shard* shards, Result* out, std::string& err, Pass pass = {}) {
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    std::vector<jtb_lk_shard> full(std::max(h->n_shards, 1));
    jtb_lk_result res;
    if (int rc = run_witness(st, ev0, ev1, h, max_nodes, max_rounds, max_repairs, max_lifts, flags, commit_read,
                             full.data(), &res, pass, err))
        return rc;
    for (int32_t s = 0; s < h->n_shards; ++s) memcpy(&shards[s], &full[s], sizeof(Shard));
    memcpy(out, &res, offsetof(Result, seconds_kernel));
    out->seconds_kernel = res.seconds_kernel;
    out->seconds_total = res.seconds_total;
    return 0;
}

}  // namespace jtb
