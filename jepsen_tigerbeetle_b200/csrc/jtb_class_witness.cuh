// jtb_class_witness.cuh — K16: the class witness (K15's lifted serial witness, then a class pass on the shards it
// leaves unproved, in which interchangeable crashed transfers are handed out earliest first) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K16 class witness").  K15 runs unchanged (run_repairs with CwPass as its
// pass): pre snapshots K12's owners and owned counters after tp_finals; post runs the class pass on every shard K15
// leaves UNKNOWN with cause UNDECIDED, NO_WITNESS or REAL_TIME, from the snapshot:
//   - the classes, once: cw_keys, a thread per transfer, keys the crashed, windowed, unowned transfers of those shards
//     by (shard, debit, credit, amount, M, A, invocation, id); one cub radix sort; cw_heads and a cub sum number the
//     classes, and cw_classes gives each member its class and each class its first sorted position;
//   - sw_init (K13's) fixes the gaps with Delta' = 0; then the class rounds, Jacobi.  cw_gaps, a warp per unfixed gap,
//     is sw_solve over sw_gaps' gather with CwCap, which drops a crashed candidate once cap members of its class are
//     gathered (the members already gathered are counted by class, a batch's lanes among themselves with
//     __match_any_sync); the solution stays in K12's poss rows and the :ok transfers take the smallest choosing gap;
//   - the hand-out: cw_un, a cub scan by class and cw_compact list each class's unowned members in order; cw_emit, a
//     thread per gap, writes one record (class << 32 | gap) per chosen member at its cub-scanned offset and checks
//     K13's rule for the :ok transfers; a cub radix sort of the records and a cub scan by class give each record its
//     rank; cw_check, a thread per record, looks up the member at that rank and its eligibility, and the smallest
//     failing gap of each class; cw_fix, a thread per gap, fixes the gaps before every failure of their classes;
//     cw_own, a thread per record, gives the members to the gaps fixed.  The host reads one 8-byte pair per round (the
//     gaps left, and the records of the next round, whose searches run before the read);
//   - K13's real time, re-sum and commit_read (sw_tgap .. sw_commit) on the shards the rounds left live.
// The decision, node counts, rounds, class rounds, members handed out and commit_read equal the CW_SEARCH CPU test
// oracle's.
#pragma once
#include "jtb_lifted_witness.cuh"

namespace jtb {

// a transfer's sort key: its class (shard .. A), then its order in the class; shard 0xffffffff: not a member
struct CwKey {
    uint32_t shard, debit, credit, amount, M, A, inv;
    uint64_t id;
};
struct CwKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, uint32_t&, uint32_t&, uint32_t&, uint32_t&, uint32_t&,
                                           uint32_t&, uint64_t&>
    operator()(CwKey& k) const {
        return {k.shard, k.debit, k.credit, k.amount, k.M, k.A, k.inv, k.id};
    }
};

struct CwDev {
    const int32_t* cls = nullptr;       // [n_t] the transfer's class, -1 none
    const int32_t* chead = nullptr;     // [classes] the class's first sorted position
    const int32_t* cun = nullptr;       // [classes] this round: unowned members
    const int32_t* cmem = nullptr;      // [members] this round: each class's unowned members from chead, in order
    int32_t* pc = nullptr;              // [m] this round: the crashed transfers the gap chose
    uint8_t* okc = nullptr;             // [m] this round: no smaller gap chose one of the gap's :ok transfers
    uint8_t* nfix = nullptr;            // [m] this round: the gap was fixed
    int32_t* cfail = nullptr;           // [classes] this round: the smallest failing gap that drew from the class
    int32_t* crounds = nullptr;         // [n_shards] class rounds that ran a gap of the shard
    int32_t* handed = nullptr;          // [n_shards] members handed to fixed gaps
};

// rg_gather's cap for the class rounds: a crashed candidate of class c passes while fewer than cap = min over its
// observed keys of floor(Delta'_k / amount) members of c are gathered before it (the earlier batches' by their
// class, this batch's lower lanes by __match_any_sync)
struct CwCap {
    const RgWarp& G;
    const int32_t* cls;
    int lane;
    __device__ __forceinline__ bool operator()(bool valid, int32_t t, int32_t a, int16_t jd, int16_t jc,
                                               int32_t n) const {
        __syncwarp();   // the earlier batches' G.ct
        const int32_t c = valid ? cls[t] : -1;
        const unsigned same = __match_any_sync(0xffffffffu, c);
        if (c < 0) return valid;
        int64_t cap = LLONG_MAX;
        if (jd >= 0) cap = G.x.d[jd] / a;
        if (jc >= 0) cap = min(cap, G.x.d[jc] / a);
        int64_t had = __popc(same & ((1u << lane) - 1));
        for (int32_t j = 0, e = min(n, JTB_RG_MAX_GATHER); j < e && had < cap; ++j) had += cls[G.ct[j]] == c;
        return had < cap;
    }
};

// thread per transfer: the sort key and the transfer
__global__ void cw_keys(RgDev d, TpDev p, const uint8_t* __restrict__ cok, CwKey* __restrict__ key,
                        int32_t* __restrict__ perm) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t];
    CwKey k;
    memset(&k, 0, sizeof k);
    k.shard = 0xffffffffu;
    if (cok[s] && p.t_fate[t] != JTB_T_OK && (p.flag[t] & TP_WIN) && p.owner[t] == RG_NONE) {
        const int32_t* q = d.t_rec + 3 * t;
        k.shard = (uint32_t)s;
        k.debit = (uint32_t)q[0];
        k.credit = (uint32_t)q[1];
        k.amount = (uint32_t)q[2];
        k.M = (uint32_t)d.t_M[t];
        k.A = (uint32_t)(d.t_A[t] + 1);
        k.inv = (uint32_t)p.t_inv[t];
        k.id = (uint64_t)d.t_id[t] ^ 0x8000000000000000ull;
    }
    key[t] = k;
    perm[t] = (int32_t)t;
}

// thread per sorted position: 1 where a class starts; *nm counts the members
__global__ void cw_heads(int32_t n_t, const CwKey* __restrict__ key, int32_t* __restrict__ head, int32_t* nm) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n_t) return;
    const CwKey& k = key[j];
    bool h = false;
    if (k.shard != 0xffffffffu) {
        atomicAdd(nm, 1);
        const CwKey* b = j > 0 ? &key[j - 1] : nullptr;
        h = !b || b->shard != k.shard || b->debit != k.debit || b->credit != k.credit || b->amount != k.amount ||
            b->M != k.M || b->A != k.A;
    }
    head[j] = h;
}

// thread per member (sorted position j < members): its class (the inclusive sum of the heads, less one)
__global__ void cw_classes(int32_t nm, const int32_t* __restrict__ perm, const int32_t* __restrict__ head,
                           const int32_t* __restrict__ cno, int32_t* __restrict__ cls, int32_t* __restrict__ mcls,
                           int32_t* __restrict__ chead) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= nm) return;
    const int32_t c = cno[j] - 1;
    cls[perm[j]] = c;
    mcls[j] = c;
    if (head[j]) chead[c] = (int32_t)j;
}

// warp per unfixed gap of a live shard: sw_gaps' gather with the class cap, and one search; the crashed transfers it
// chose are counted into c.pc and *nrec
__global__ void __launch_bounds__(RG_WARPS * 32) cw_gaps(RgDev d, TpDev p, SwDev w, CwDev c, int32_t* nrec) {
    __shared__ RgWarp smem[RG_WARPS];
    const int lane = threadIdx.x & 31;
    RgWarp& G = smem[threadIdx.x >> 5];
    const int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (wi >= d.m || w.fixed[wi]) return;
    const int32_t i = (int32_t)wi, s = d.shard[d.ord[i]];
    int64_t nodes = 0;
    int32_t chosen = 0;
    const bool ok = sw_solve(d, p, w, G, lane, i, [&](int32_t t) {
        return (p.flag[t] & TP_WIN) && p.lo[t] <= i && i <= p.hi[t] && p.owner[t] == RG_NONE;
    }, nodes, chosen, CwCap{G, c.cls, lane});
    const int32_t* ps = p.poss + (int64_t)i * JTB_TP_MAX_GATHER;
    int32_t ncr = 0;
    __syncwarp();
    for (int32_t base = 0; base < chosen; base += 32) {
        const int32_t k = base + lane;
        ncr += __popc(__ballot_sync(0xffffffffu, k < chosen && p.t_fate[ps[k]] != JTB_T_OK));
    }
    if (lane != 0) return;
    atomicAdd(&w.cnt[(int64_t)s * SW_COUNTERS + 3], (unsigned long long)nodes);
    atomicMax(&c.crounds[s], w.round + 1);
    p.pn[i] = chosen;
    c.pc[i] = ncr;
    if (ncr) atomicAdd(nrec, ncr);
    if (!ok) atomicMin(&w.sfail[s], i);
}

// thread per member: 1 while no gap owns it
__global__ void cw_un(int32_t nm, const int32_t* __restrict__ perm, const int32_t* __restrict__ owner,
                      int32_t* __restrict__ un) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j < nm) un[j] = owner[perm[j]] == RG_NONE;
}

// thread per member: the unowned ones, by their rank in the class (ur, the scan of un by class), from chead
__global__ void cw_compact(int32_t nm, const int32_t* __restrict__ perm, const int32_t* __restrict__ mcls,
                           const int32_t* __restrict__ un, const int32_t* __restrict__ ur, CwDev c, int32_t* cmem,
                           int32_t* cun) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= nm || !un[j]) return;
    cmem[c.chead[mcls[j]] + ur[j]] = perm[j];
    atomicAdd(&cun[mcls[j]], 1);
}

// thread per unfixed gap: K13's rule for its :ok transfers, and a record per crashed transfer it chose at roff[i]
__global__ void cw_emit(int32_t m, TpDev p, SwDev w, CwDev c, const int32_t* __restrict__ roff,
                        unsigned long long* __restrict__ rec, int32_t* __restrict__ ones) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m || w.fixed[i]) return;
    const int32_t n = p.pn[i];
    const int32_t* ps = p.poss + i * JTB_TP_MAX_GATHER;
    bool ok = true;
    for (int32_t k = 0, at = roff[i]; k < n; ++k) {
        const int32_t t = ps[k];
        if (p.t_fate[t] == JTB_T_OK) {
            ok &= w.cmin[t] == i;
        } else {
            rec[at] = (unsigned long long)(uint32_t)c.cls[t] << 32 | (uint32_t)i;
            ones[at++] = 1;
        }
    }
    c.okc[i] = ok;
}

struct CwSameClass {
    __device__ __forceinline__ bool operator()(unsigned long long a, unsigned long long b) const {
        return (a >> 32) == (b >> 32);
    }
};

// thread per record (sorted by class, then gap): the member at its rank, when it exists and is eligible for the gap
// and the gap keeps K13's rule; otherwise the gap fails the class
__global__ void cw_check(int32_t nrec, RgDev d, TpDev p, CwDev c, const unsigned long long* __restrict__ rec,
                         const int32_t* __restrict__ rank, int32_t* __restrict__ rt) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= nrec) return;
    const int32_t cl = (int32_t)(rec[k] >> 32), g = (int32_t)(uint32_t)rec[k], r = rank[k];
    int32_t t = -1;
    if (c.okc[g] && r < c.cun[cl]) {
        t = c.cmem[c.chead[cl] + r];
        const int32_t u = d.ord[g], s = d.shard[u], cp = d.comp[u];
        const int32_t lower = g > 0 && d.shard[d.ord[g - 1]] == s ? d.ord[g - 1] : -1;
        const int32_t ivl = lower >= 0 ? d.inv[lower] : -1;
        if (!((p.flag[t] & TP_WIN) && p.lo[t] <= g && g <= p.hi[t] && p.t_inv[t] < cp && d.t_A[t] < cp &&
              !(d.t_M[t] < ivl)))
            t = -1;
    }
    rt[k] = t;
    if (t < 0) atomicMin(&c.cfail[cl], g);
}

// thread per unfixed gap: fixed when it keeps K13's rule and comes before every failure of the classes it drew from;
// then it owns its :ok transfers (cw_own gives it its members); the gaps of a failed shard stop
__global__ void cw_fix(int32_t m, RgDev d, TpDev p, SwDev w, CwDev c) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m || w.fixed[i]) return;
    c.nfix[i] = 0;
    if (w.sfail[d.shard[d.ord[i]]] != RG_NONE) { w.fixed[i] = 1; return; }
    const int32_t n = p.pn[i];
    const int32_t* ps = p.poss + i * JTB_TP_MAX_GATHER;
    bool fix = c.okc[i];
    for (int32_t k = 0; k < n && fix; ++k)
        if (p.t_fate[ps[k]] != JTB_T_OK) fix = i < c.cfail[c.cls[ps[k]]];
    if (!fix) { atomicAdd(w.unfixed, 1); return; }
    for (int32_t k = 0; k < n; ++k)
        if (p.t_fate[ps[k]] == JTB_T_OK) p.owner[ps[k]] = (int32_t)i;
    w.fixed[i] = 1;
    c.nfix[i] = 1;
}

// thread per record: the member goes to its gap when the gap was fixed
__global__ void cw_own(int32_t nrec, RgDev d, TpDev p, CwDev c, const unsigned long long* __restrict__ rec,
                       const int32_t* __restrict__ rt) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= nrec) return;
    const int32_t g = (int32_t)(uint32_t)rec[k];
    if (!c.nfix[g]) return;
    p.owner[rt[k]] = g;
    atomicAdd(&c.handed[d.shard[d.ord[g]]], 1);
}

// ---- host ---------------------------------------------------------------------------------------------------------

// K16's pass over K15's results (run_repairs' Pass)
struct CwPass {
    int32_t* owner0 = nullptr;   // K12's owners and owned counters, as tp_finals left them
    int64_t* own0 = nullptr;

    int pre(cudaStream_t st, TpStage& g, std::string& err) {
        JTB_OK(g.A.alloc(&owner0, g.nT)); JTB_OK(g.A.alloc(&own0, g.cells));
        JTB_OK(cudaMemcpyAsync(owner0, g.p.owner, (size_t)g.nT * 4, cudaMemcpyDeviceToDevice, st));
        JTB_OK(cudaMemcpyAsync(own0, g.own, (size_t)g.cells * 8, cudaMemcpyDeviceToDevice, st));
        return 0;
    }

    int post(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, TpStage& g, int32_t max_rounds,
             jtb_cw_shard* shards, std::vector<int32_t>& cr_h, float& ms, std::string& err) {
        const int32_t S = g.S, nT = g.nT, m = g.m;
        const TlHost& T = g.T;
        std::vector<uint8_t> cok(S, 0);
        bool any = false;
        for (int32_t s = 0; s < S; ++s) {
            const jtb_cw_shard& o = shards[s];
            any |= (cok[s] = g.dev[s] && o.valid == JTB_UNKNOWN &&
                             (o.cause == JTB_CAUSE_UNDECIDED || o.cause == JTB_CAUSE_NO_WITNESS ||
                              o.cause == JTB_CAUSE_REAL_TIME));
        }
        if (!any) return 0;
        CallAllocs& A = g.A;
        RgDev& x = g.x;
        TpDev& p = g.p;
        JTB_OK(cudaMemcpyAsync(p.owner, owner0, (size_t)nT * 4, cudaMemcpyDeviceToDevice, st));
        JTB_OK(cudaMemcpyAsync(g.own, own0, (size_t)g.cells * 8, cudaMemcpyDeviceToDevice, st));
        SwDev w;
        CwDev c;
        w.t_okcomp = g.d.t_okcomp;
        std::vector<int32_t> rd_cidx(m);
        for (int32_t i = 0; i < m; ++i) rd_cidx[i] = h->index[g.H.r_ev[g.d_of[i]]];
        const int32_t* d_cidx;
        int32_t *d_cr, *perm0, *perm, *head, *cno, *cls, *mcls, *chead, *un, *ur, *cmem, *cun, *roff, *words;
        CwKey *key0, *key;
        uint8_t* stmp;
        JTB_OK(A.put(&w.sok, cok, st)); JTB_OK(A.put(&d_cidx, rd_cidx, st));
        JTB_OK(A.alloc(&w.fixed, m)); JTB_OK(A.alloc(&w.cmin, nT)); JTB_OK(A.alloc(&w.sfail, S));
        JTB_OK(A.alloc(&w.sunf, S)); JTB_OK(A.alloc(&w.unfixed, 1)); JTB_OK(A.alloc(&w.cnt, (size_t)S * SW_COUNTERS));
        JTB_OK(A.alloc(&w.gmax, m)); JTB_OK(A.alloc(&w.gmin, m)); JTB_OK(A.alloc(&w.skey, m));
        JTB_OK(A.alloc(&w.x, m)); JTB_OK(A.alloc(&w.P, m)); JTB_OK(A.alloc(&w.rtkey, S)); JTB_OK(A.alloc(&w.rtid, S));
        JTB_OK(A.alloc(&w.bad, 1)); JTB_OK(A.alloc(&d_cr, nT));
        JTB_OK(A.alloc(&key0, nT)); JTB_OK(A.alloc(&key, nT)); JTB_OK(A.alloc(&perm0, nT)); JTB_OK(A.alloc(&perm, nT));
        JTB_OK(A.alloc(&head, nT)); JTB_OK(A.alloc(&cno, nT)); JTB_OK(A.alloc(&cls, nT)); JTB_OK(A.alloc(&mcls, nT));
        JTB_OK(A.alloc(&chead, nT)); JTB_OK(A.alloc(&un, nT)); JTB_OK(A.alloc(&ur, nT)); JTB_OK(A.alloc(&cmem, nT));
        JTB_OK(A.alloc(&cun, nT)); JTB_OK(A.alloc(&c.cfail, nT)); JTB_OK(A.alloc(&roff, m));
        JTB_OK(A.alloc(&c.pc, m)); JTB_OK(A.alloc(&c.okc, m)); JTB_OK(A.alloc(&c.nfix, m));
        JTB_OK(A.alloc(&c.crounds, S)); JTB_OK(A.alloc(&c.handed, S)); JTB_OK(A.alloc(&words, 4));
        c.cls = cls; c.chead = chead; c.cun = cun; c.cmem = cmem;
        // the records of a round: sorted keys, their ranks and members; grown as a round needs
        int64_t rec_cap = 0;
        unsigned long long *rec0 = nullptr, *rec = nullptr;
        int32_t *ones = nullptr, *rank = nullptr, *rt = nullptr;
        auto grow = [&](int64_t need) -> cudaError_t {
            if (need <= rec_cap) return cudaSuccess;
            rec_cap = std::max<int64_t>(need, 2 * rec_cap);
            cudaError_t e;
            if ((e = A.alloc(&rec0, rec_cap)) != cudaSuccess || (e = A.alloc(&rec, rec_cap)) != cudaSuccess ||
                (e = A.alloc(&ones, rec_cap)) != cudaSuccess || (e = A.alloc(&rank, rec_cap)) != cudaSuccess)
                return e;
            return A.alloc(&rt, rec_cap);
        };
        JTB_OK(grow(std::max<int64_t>(nT, 16)));
        // cub's temporary storage: the largest of its uses at their largest sizes
        size_t stmp_bytes = 0, b = 0;
        auto need = [&](cudaError_t e) {
            stmp_bytes = std::max(stmp_bytes, b);
            return e;
        };
        JTB_OK(need(cub::DeviceScan::InclusiveScanByKey(nullptr, b, w.skey, w.x, w.P, MaxOp{}, m,
                                                        cuda::std::equal_to<>{}, st)));
        JTB_OK(need(cub::DeviceRadixSort::SortPairs(nullptr, b, key0, key, perm0, perm, nT, CwKeyDecomposer{}, st)));
        JTB_OK(need(cub::DeviceScan::InclusiveSum(nullptr, b, head, cno, nT, st)));
        JTB_OK(need(cub::DeviceScan::ExclusiveScanByKey(nullptr, b, mcls, un, ur, cuda::std::plus<>{}, 0, nT,
                                                        cuda::std::equal_to<>{}, st)));
        JTB_OK(need(cub::DeviceScan::ExclusiveSum(nullptr, b, c.pc, roff, m, st)));
        JTB_OK(A.alloc(&stmp, stmp_bytes));
        size_t rec_bytes = 0;   // the records' sort and scan, sized per round
        uint8_t* rtmp = nullptr;
        auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };
        // the classes
        int32_t nm = 0;
        JTB_OK(cudaMemsetAsync(words, 0, 16, st));
        JTB_OK(cudaMemsetAsync(cls, 0xff, (size_t)nT * 4, st));   // -1
        size_t tb;
        if (nT > 0) {
            cw_keys<<<grid(nT, 256), 256, 0, st>>>(x, p, w.sok, key0, perm0);
            tb = stmp_bytes;
            JTB_OK(cub::DeviceRadixSort::SortPairs(stmp, tb, key0, key, perm0, perm, nT, CwKeyDecomposer{}, st));
            cw_heads<<<grid(nT, 256), 256, 0, st>>>(nT, key, head, words);
            tb = stmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveSum(stmp, tb, head, cno, nT, st));
            JTB_OK(cudaMemcpyAsync(&nm, words, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            if (nm > 0) cw_classes<<<grid(nm, 256), 256, 0, st>>>(nm, perm, head, cno, cls, mcls, chead);
        }
        JTB_OK(cudaMemsetAsync(w.sfail, 0x7f, (size_t)S * 4, st));   // RG_NONE
        JTB_OK(cudaMemsetAsync(w.sunf, 0x7f, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(w.cnt, 0, (size_t)S * SW_COUNTERS * 8, st));
        JTB_OK(cudaMemsetAsync(w.unfixed, 0, 4, st));
        JTB_OK(cudaMemsetAsync(c.crounds, 0, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(c.handed, 0, (size_t)S * 4, st));
        sw_init<<<grid(m, 256), 256, 0, st>>>(x, p, w);
        int32_t unfixed = 0;
        JTB_OK(cudaMemcpyAsync(&unfixed, w.unfixed, 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        // the class rounds; a round's searches run before the host reads the previous round's gaps left
        auto search = [&](int32_t r) -> int {
            JTB_OK(cudaMemsetAsync(w.cmin, 0x7f, (size_t)nT * 4, st));
            JTB_OK(cudaMemsetAsync(c.pc, 0, (size_t)m * 4, st));
            JTB_OK(cudaMemsetAsync(words + 1, 0, 4, st));
            w.round = r;
            cw_gaps<<<grid(m, RG_WARPS), RG_WARPS * 32, 0, st>>>(x, p, w, c, words + 1);
            return 0;
        };
        int32_t hw[2] = {unfixed, 0};   // the gaps left, the records of the round that searched
        if (unfixed > 0 && max_rounds > 0) {
            if (int rc = search(0)) return rc;
            JTB_OK(cudaMemcpyAsync(hw + 1, words + 1, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
        }
        for (int32_t r = 0; hw[0] > 0 && r < max_rounds; ++r) {
            const int32_t nrec = hw[1];
            // the unowned members of every class, in order
            if (nm > 0) {
                JTB_OK(cudaMemsetAsync(cun, 0, (size_t)nm * 4, st));
                cw_un<<<grid(nm, 256), 256, 0, st>>>(nm, perm, p.owner, un);
                tb = stmp_bytes;
                JTB_OK(cub::DeviceScan::ExclusiveScanByKey(stmp, tb, mcls, un, ur, cuda::std::plus<>{}, 0, nm,
                                                           cuda::std::equal_to<>{}, st));
                cw_compact<<<grid(nm, 256), 256, 0, st>>>(nm, perm, mcls, un, ur, c, cmem, cun);
            }
            // the records, their ranks, and the checks
            JTB_OK(grow(nrec));
            tb = stmp_bytes;
            JTB_OK(cub::DeviceScan::ExclusiveSum(stmp, tb, c.pc, roff, m, st));
            cw_emit<<<grid(m, 256), 256, 0, st>>>(m, p, w, c, roff, rec0, ones);
            if (nrec > 0) {
                size_t nb = 0, sb = 0;
                JTB_OK(cub::DeviceRadixSort::SortKeys(nullptr, nb, rec0, rec, nrec, 0, 64, st));
                JTB_OK(cub::DeviceScan::ExclusiveScanByKey(nullptr, sb, rec, ones, rank, cuda::std::plus<>{}, 0, nrec,
                                                           CwSameClass{}, st));
                if (std::max(nb, sb) > rec_bytes) {
                    rec_bytes = std::max(nb, sb);
                    JTB_OK(A.alloc(&rtmp, rec_bytes));
                }
                nb = rec_bytes;
                JTB_OK(cub::DeviceRadixSort::SortKeys(rtmp, nb, rec0, rec, nrec, 0, 64, st));
                sb = rec_bytes;
                JTB_OK(cub::DeviceScan::ExclusiveScanByKey(rtmp, sb, rec, ones, rank, cuda::std::plus<>{}, 0, nrec,
                                                           CwSameClass{}, st));
                JTB_OK(cudaMemsetAsync(c.cfail, 0x7f, (size_t)std::max(nm, 1) * 4, st));
                cw_check<<<grid(nrec, 256), 256, 0, st>>>(nrec, x, p, c, rec, rank, rt);
            }
            JTB_OK(cudaMemsetAsync(w.unfixed, 0, 4, st));
            cw_fix<<<grid(m, 256), 256, 0, st>>>(m, x, p, w, c);
            if (nrec > 0) cw_own<<<grid(nrec, 256), 256, 0, st>>>(nrec, x, p, c, rec, rt);
            if (r + 1 < max_rounds)
                if (int rc = search(r + 1)) return rc;
            JTB_OK(cudaGetLastError());
            JTB_OK(cudaMemcpyAsync(hw, w.unfixed, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaMemcpyAsync(hw + 1, words + 1, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
        }
        if (hw[0] > 0) sw_unfixed<<<grid(m, 256), 256, 0, st>>>(m, x, w);
        // real time and the counters, as K13
        JTB_OK(cudaMemsetAsync(w.gmax, 0x80, (size_t)m * 4, st));   // INT_MIN
        JTB_OK(cudaMemsetAsync(w.gmin, 0x7f, (size_t)m * 4, st));   // > every position
        JTB_OK(cudaMemsetAsync(w.rtkey, 0xff, (size_t)S * 8, st));
        JTB_OK(cudaMemsetAsync(w.rtid, 0xff, (size_t)S * 8, st));
        JTB_OK(cudaMemsetAsync(w.bad, 0, 4, st));
        JTB_OK(cudaMemsetAsync(g.own, 0, (size_t)g.cells * 8, st));
        if (nT > 0) sw_tgap<<<grid(nT, 256), 256, 0, st>>>(x, p, w);
        sw_scan_in<<<grid(m, 256), 256, 0, st>>>(x, w);
        tb = stmp_bytes;
        JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, w.skey, w.x, w.P, MaxOp{}, m, cuda::std::equal_to<>{}, st));
        sw_rt<<<grid(m, 256), 256, 0, st>>>(x, p, w);
        sw_sum<<<grid((int64_t)m * 32, 256), 256, 0, st>>>(x, p, w);
        if (nT > 0) {
            sw_after<<<grid(nT, 256), 256, 0, st>>>(x, p, w);
            sw_commit<<<grid(nT, 256), 256, 0, st>>>(x, p, w, d_cidx, d_cr);
        }
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<unsigned long long> cnt_h((size_t)S * SW_COUNTERS), rtkey_h(S);
        std::vector<int32_t> sfail_h(S), sunf_h(S), cr_rounds(S), handed_h(S), dcr(nT);
        unsigned int bad = 0;
        JTB_OK(cudaMemcpyAsync(cnt_h.data(), w.cnt, cnt_h.size() * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(rtkey_h.data(), w.rtkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(sfail_h.data(), w.sfail, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(sunf_h.data(), w.sunf, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(cr_rounds.data(), c.crounds, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(handed_h.data(), c.handed, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(&bad, w.bad, 4, cudaMemcpyDeviceToHost, st));
        if (nT > 0) JTB_OK(cudaMemcpyAsync(dcr.data(), d_cr, (size_t)nT * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        if (bad) { err = "the counters of a serial witness do not add up"; return -1; }
        for (int32_t s = 0; s < S; ++s) {
            if (!cok[s]) continue;
            jtb_cw_shard& o = shards[s];
            const unsigned long long* cc = &cnt_h[(size_t)s * SW_COUNTERS];
            o.nodes += (int64_t)cc[3];
            o.class_rounds = cr_rounds[s];
            o.n_handed = handed_h[s];
            if (sfail_h[s] != RG_NONE || sunf_h[s] != RG_NONE) {
                o.class_cause = JTB_CAUSE_NO_WITNESS;
            } else if (rtkey_h[s] != ~0ull) {
                o.class_cause = JTB_CAUSE_REAL_TIME;
            } else {
                o.valid = JTB_VALID;
                o.cause = 0;
                o.fail_index = -1;
                o.transfer_id = -1;
                o.n_committed = (int64_t)cc[0];
                o.n_committed_crashed = (int64_t)cc[1];
                o.n_after = (int64_t)cc[2];
                for (int32_t t = T.t_off[s]; t < T.t_off[s + 1]; ++t) cr_h[t] = dcr[t];
            }
        }
        return 0;
    }
};

inline int run_class_witness(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                             int64_t max_nodes, int32_t max_rounds, int32_t max_repairs, int32_t max_lifts,
                             int32_t flags, int32_t* commit_read, jtb_cw_shard* shards, jtb_cw_result* out,
                             std::string& err) {
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    return run_repairs(st, ev0, ev1, h, max_nodes, max_rounds, max_repairs, max_lifts, commit_read, shards, out, flags,
                       err, CwPass{});
}

}  // namespace jtb
