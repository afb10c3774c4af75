// jtb_lookup_witness.cuh — K17: the lookup witness (K16's class witness, then every :ok lookup of a shard it proves is
// placed in the shard's serial order and the merged order is checked) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K17 lookup witness").  K16 runs unchanged (run_repairs with LkPass, which
// runs CwPass and then the lookup pass).  The lookup pass works on the shards K16 proves that have an :ok lookup:
//   - lk_shown, a thread per record: the transfers some lookup returns; lk_gap, a thread per transfer: the commit gap
//     G(t) (a global position; rs_off[s + 1] is "after the last read") from K16's owners, a count per (shard, G) and
//     D_g's largest invocation; a cub sum and K13's max-scan by shard give N(g) and the reads' points Q;
//   - lk_linit, a thread per lookup, starts lo at the shard's first gap; lk_rec, a thread per record in K9's (lookup, id) order: records that name no transfer, differ from it, repeat an
//     id or name a transfer that never commits, and lo = max G; lk_below, the records below lo; lk_place, a thread per
//     lookup: lo <= hi (the records below lo are all the committed transfers below lo), hi and the position by binary
//     searches of N and Q, and the shown part a of D_g;
//   - the chain test: a cub sort of the lookups by (position, a, lookup), lk_heads and a max-scan (each group's start),
//     lk_layer (thread per record: a transfer's layer is the first lookup of its gap that returns it), lk_lcount and a
//     cub sum (transfers per layer), lk_chain (thread per lookup: the transfers at or below its layer are exactly a);
//   - the merged order: lk_ops keys every read, committed transfer and lookup by (position, layer, invocation); one cub
//     radix sort; lk_scan_in and cub's InclusiveScanByKey (max, by shard); lk_rt, the first op whose point is not below
//     its completion; lk_rt_lookup, the last lookup at or before it;
//   - the outputs, all on the device: lk_fail_index (thread per shard: the lookup that fails), lk_lookup_read (thread
//     per lookup) and lk_after (thread per transfer: the crashed transfers committed after the last read).
// The decision, commit_read and lookup_read equal the LK_SEARCH CPU test oracle's.
#pragma once
#include "jtb_class_witness.cuh"

namespace jtb {

struct LkKey {   // a lookup in the chain test: (shard position, shown part of D_g, lookup); 0xffffffff: not placed
    uint32_t gp, a, l;
};
struct LkKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, uint32_t&, uint32_t&> operator()(LkKey& k) const {
        return {k.gp, k.a, k.l};
    }
};
struct LkOpKey {   // an op of the merged order: (shard position, layer, invocation + 1); 0xffffffff: not in it
    uint32_t gp, sub, iv;
};
struct LkOpKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, uint32_t&, uint32_t&> operator()(LkOpKey& k) const {
        return {k.gp, k.sub, k.iv};
    }
};

constexpr int32_t LK_NEVER = INT_MAX;   // G of a transfer that never commits

struct LkDev {
    const uint8_t* on = nullptr;        // [n_shards] K16 VALID with an :ok lookup
    const uint8_t* cls = nullptr;       // [n_shards] K16's class pass ran (its owners are in p.owner)
    const int32_t* kowner = nullptr;    // [n_t] the owners K15 ended with
    const int32_t* l_inv = nullptr;     // [n_l]
    uint8_t* shown = nullptr;           // [n_t]
    int32_t* G = nullptr;               // [n_t] commit gap, LK_NEVER none
    int32_t* layer = nullptr;           // [n_t] the sorted rank of the first lookup of its gap returning it, RG_NONE
    int32_t* cum = nullptr;             // [m + n_shards] committed transfers with G + s <= index (inclusive sum)
    const int32_t* Q = nullptr;         // [m] K13's point of the read at each position
    int32_t* lo = nullptr;              // [n_l]
    int32_t* below = nullptr;           // [n_l] records with G < lo
    uint8_t* bad = nullptr;             // [n_l] an unplaceable record
    int32_t* lpos = nullptr;            // [n_l] the position
    int32_t* la = nullptr;              // [n_l] the shown part of D_g
    int32_t* grank = nullptr;           // [n_l] the sorted rank in the chain test
    int32_t* gstart = nullptr;          // [n_l] by sorted rank: its group's first rank
    int32_t* lfail = nullptr;           // [n_shards] the smallest unplaceable lookup, RG_NONE none
    int32_t* cfail = nullptr;           // [n_shards] the smallest lookup that breaks the chain, RG_NONE none
    int32_t* rfail = nullptr;           // [n_shards] the first op of the merged order that breaks real time
    int32_t* rlast = nullptr;           // [n_shards] the last lookup at or before it, -1 none
    int32_t* rfirst = nullptr;          // [n_shards] the shard's first lookup in the merged order, INT_MAX none
};

__device__ __forceinline__ int32_t lk_end(const TpDev& p, int32_t s) { return p.rs_off[s + 1]; }

// thread per record: the transfer it names is shown
__global__ void lk_shown(TlDev d, LkDev k) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= d.n_rec) return;
    const int32_t l = tl_lookup_of(d, g), slot = d.rec_slot[g];
    if (k.on[d.l_shard[l]] && slot >= 0) k.shown[d.tperm[slot]] = 1;
}

// thread per transfer: G, the count per (shard, G) and D_g's largest invocation
__global__ void lk_gap(TpDev p, LkDev k, int32_t* __restrict__ hist, int32_t* __restrict__ gmax) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t];
    if (!k.on[s]) return;
    const int32_t o = k.cls[s] ? p.owner[t] : k.kowner[t], f = p.t_fate[t], end = lk_end(p, s);
    const int32_t G = o != RG_NONE ? o : f == JTB_T_OK || (f != JTB_T_FAIL && k.shown[t]) ? end : LK_NEVER;
    k.G[t] = G;
    if (G == LK_NEVER) return;
    atomicAdd(&hist[G + s], 1);
    if (G < end) atomicMax(&gmax[G], p.t_inv[t]);
}

// committed transfers of shard s with G < g
__device__ __forceinline__ int32_t lk_nlt(const TpDev& p, const LkDev& k, int32_t s, int32_t g) {
    const int32_t base = p.rs_off[s] + s;
    return g + s > base ? k.cum[g + s - 1] - (base > 0 ? k.cum[base - 1] : 0) : 0;
}

// thread per record in (lookup, id) order: the unplaceable records and lo
__global__ void lk_rec(TlDev d, TpDev p, LkDev k) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.n_rec) return;
    const TlRKey key = d.rkey[i];
    const int32_t l = (int32_t)key.lookup, s = d.l_shard[l];
    if (!k.on[s]) return;
    const int32_t g = d.rval[i], slot = d.rec_slot[g];
    bool bad = slot < 0 || (i > 0 && d.rkey[i - 1].lookup == key.lookup && d.rkey[i - 1].idu == key.idu);
    if (!bad) {
        const int32_t t = d.tperm[slot];
        const int32_t* r = tl_rec(d, l, g);
        const int32_t* q = d.t_rec + 3 * (int64_t)t;
        bad = q[0] != r[2] || q[1] != r[3] || q[2] != r[4] || k.G[t] == LK_NEVER;
        if (!bad) atomicMax(&k.lo[l], k.G[t]);
    }
    if (bad) k.bad[l] = 1;
}

// thread per record: the records below lo
__global__ void lk_below(TlDev d, LkDev k) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= d.n_rec) return;
    const int32_t l = tl_lookup_of(d, g), slot = d.rec_slot[g];
    if (!k.on[d.l_shard[l]] || k.bad[l] || slot < 0) return;
    if (k.G[d.tperm[slot]] < k.lo[l]) atomicAdd(&k.below[l], 1);
}

// thread per lookup: the range [lo, hi], the position and the shown part of D_g; the chain test's sort key
__global__ void lk_place(TlDev d, TpDev p, LkDev k, LkKey* __restrict__ key, int32_t* __restrict__ perm) {
    const int64_t li = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (li >= d.n_l) return;
    const int32_t l = (int32_t)li, s = d.l_shard[l];
    key[l] = LkKey{0xffffffffu, 0, (uint32_t)l};
    perm[l] = l;
    if (!k.on[s]) return;
    const int32_t lo = k.lo[l], n0 = p.rs_off[s], end = lk_end(p, s);
    const int32_t cnt = (int32_t)(d.rec_base[l + 1] - d.rec_base[l]);
    if (k.bad[l] || k.below[l] != lk_nlt(p, k, s, lo)) { atomicMin(&k.lfail[s], l); return; }
    // hi: the first g with N(g) > cnt, else end
    const int32_t base = n0 + s, sub = base > 0 ? k.cum[base - 1] : 0;
    int32_t a = base, b = end + s + 1;
    while (a < b) {
        const int32_t c = (a + b) >> 1;
        if (k.cum[c] - sub > cnt) b = c; else a = c + 1;
    }
    const int32_t hi = min(a - s, end);
    // the latest g in [lo, hi] whose lower read's point is below cp(l): Q is non-decreasing
    const int32_t cp = d.l_comp[l];
    int32_t x = lo, y = hi + 1;   // the first g in [lo, hi + 1) with Q[g - 1] >= cp
    while (x < y) {
        const int32_t c = (x + y) >> 1;
        if (c > n0 && k.Q[c - 1] >= cp) y = c; else x = c + 1;
    }
    const int32_t pos = max(lo, x - 1);
    k.lpos[l] = pos;
    k.la[l] = cnt - lk_nlt(p, k, s, pos);
    key[l] = LkKey{(uint32_t)(pos + s), (uint32_t)k.la[l], (uint32_t)l};
}

// thread per sorted lookup: its rank, and 1 where a group (one position) starts
__global__ void lk_heads(int32_t n_l, const LkKey* __restrict__ key, const int32_t* __restrict__ perm, LkDev k,
                         int32_t* __restrict__ head) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n_l) return;
    k.grank[perm[j]] = (int32_t)j;
    head[j] = j == 0 || key[j - 1].gp != key[j].gp ? (int32_t)j : 0;
}

// thread per record in (lookup, id) order: a transfer's layer is the smallest rank of a lookup of its gap returning it
__global__ void lk_layer(TlDev d, LkDev k, const uint8_t* __restrict__ live) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.n_rec) return;
    const int32_t l = (int32_t)d.rkey[i].lookup, s = d.l_shard[l], slot = d.rec_slot[d.rval[i]];
    if (!live[s] || slot < 0) return;
    const int32_t t = d.tperm[slot];
    if (k.G[t] == k.lpos[l]) atomicMin(&k.layer[t], k.grank[l]);
}

// thread per transfer: the count of each layer
__global__ void lk_lcount(int32_t n_t, LkDev k, int32_t* __restrict__ cnt) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t < n_t && k.layer[t] != RG_NONE) atomicAdd(&cnt[k.layer[t]], 1);
}

// thread per sorted lookup of a live shard: the transfers of its gap at or below its layer are exactly its shown part
__global__ void lk_chain(TlDev d, LkDev k, const int32_t* __restrict__ perm, const int32_t* __restrict__ ccum,
                         const uint8_t* __restrict__ live) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= d.n_l) return;
    const int32_t l = perm[j], s = d.l_shard[l];
    if (!live[s]) return;
    const int32_t b = k.gstart[j];
    if (ccum[j] - (b > 0 ? ccum[b - 1] : 0) != k.la[l]) atomicMin(&k.cfail[s], l);
}

// the merged order's keys: reads [0, m), transfers [m, m + n_t), lookups [m + n_t, ..)
__global__ void lk_ops(RgDev x, TlDev d, TpDev p, LkDev k, const uint8_t* __restrict__ live, LkOpKey* __restrict__ key,
                       int32_t* __restrict__ val) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t m = x.m, nT = p.n_t;
    if (e >= m + nT + d.n_l) return;
    LkOpKey q{0xffffffffu, 0, 0};
    if (e < m) {
        const int32_t u = x.ord[e], s = x.shard[u];
        if (live[s]) q = LkOpKey{(uint32_t)(e + s), 0xffffffffu, 0};
    } else if (e < m + nT) {
        const int32_t t = (int32_t)(e - m), s = p.t_shard[t], G = k.G[t];
        if (live[s] && G != LK_NEVER) {
            const int32_t ly = k.layer[t];
            const uint32_t sub = ly == RG_NONE ? 0xfffffffeu : 2u * (uint32_t)(ly - k.gstart[ly]);
            q = LkOpKey{(uint32_t)(G + s), sub, (uint32_t)(p.t_inv[t] + 1)};
        }
    } else {
        const int32_t l = (int32_t)(e - m - nT), s = d.l_shard[l];
        if (live[s]) {
            const int32_t r = k.grank[l];
            q = LkOpKey{(uint32_t)(k.lpos[l] + s), 2u * (uint32_t)(r - k.gstart[r]) + 1, 0};
        }
    }
    key[e] = q;
    val[e] = (int32_t)e;
}

// the op's shard, invocation and completion (INT_MAX: never completed :ok)
__device__ __forceinline__ void lk_op(const RgDev& x, const TlDev& d, const TpDev& p, const LkDev& k, int32_t e,
                                      int32_t& s, int32_t& iv, int32_t& cp) {
    const int32_t m = x.m, nT = p.n_t;
    if (e < m) {
        const int32_t u = x.ord[e];
        s = x.shard[u]; iv = x.inv[u]; cp = x.comp[u];
    } else if (e < m + nT) {
        const int32_t t = e - m;
        s = p.t_shard[t]; iv = p.t_inv[t]; cp = d.t_okcomp[t];
    } else {
        const int32_t l = e - m - nT;
        s = d.l_shard[l]; iv = k.l_inv[l]; cp = d.l_comp[l];
    }
}

// thread per sorted op: the scan's key and input
__global__ void lk_scan_in(int64_t n, RgDev x, TlDev d, TpDev p, LkDev k, const LkOpKey* __restrict__ key,
                           const int32_t* __restrict__ val, int32_t* __restrict__ skey, int32_t* __restrict__ xin) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n) return;
    int32_t s = -1, iv = INT_MIN, cp;
    if (key[j].gp != 0xffffffffu) lk_op(x, d, p, k, val[j], s, iv, cp);
    skey[j] = s;
    xin[j] = iv;
}

// thread per sorted op: the first op of its shard whose point is not below its completion
__global__ void lk_rt(int64_t n, RgDev x, TlDev d, TpDev p, LkDev k, const LkOpKey* __restrict__ key,
                      const int32_t* __restrict__ val, const int32_t* __restrict__ P) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n || key[j].gp == 0xffffffffu) return;
    int32_t s, iv, cp;
    lk_op(x, d, p, k, val[j], s, iv, cp);
    if (P[j] >= cp) atomicMin(&k.rfail[s], (int32_t)j);
}

// thread per sorted op: the last lookup at or before the first failing op of its shard, and its first lookup
__global__ void lk_rt_lookup(int64_t n, RgDev x, TpDev p, const TlDev d, LkDev k, const LkOpKey* __restrict__ key,
                             const int32_t* __restrict__ val) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n || key[j].gp == 0xffffffffu) return;
    const int32_t e = val[j];
    if (e < x.m + p.n_t) return;
    const int32_t s = d.l_shard[e - x.m - p.n_t];
    if (j <= k.rfail[s]) atomicMax(&k.rlast[s], (int32_t)j);
    atomicMin(&k.rfirst[s], (int32_t)j);
}

// thread per lookup: lo starts at the shard's first gap; the counters are cleared
__global__ void lk_linit(TlDev d, TpDev p, LkDev k) {
    const int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (l >= d.n_l) return;
    k.lo[l] = p.rs_off[d.l_shard[l]];
    k.below[l] = 0;
    k.bad[l] = 0;
}

// the shard is proved with its lookups placed
__device__ __forceinline__ bool lk_ok(const LkDev& k, int32_t s) {
    return k.on[s] && k.lfail[s] == RG_NONE && k.cfail[s] == RG_NONE && k.rfail[s] == RG_NONE;
}

// thread per shard with lookups: the completion :index of the lookup that fails, INT_MIN none: the smallest
// unplaceable one, else the smallest that breaks the nesting, else the last one at or before the first op that breaks
// real time (the shard's first lookup in the merged order when none precedes that op)
__global__ void lk_fail_index(int32_t S, int32_t m, int32_t n_t, LkDev k, const int32_t* __restrict__ l_cidx,
                              const int32_t* __restrict__ val, int32_t* __restrict__ fidx) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= S) return;
    int32_t l = -1;
    if (k.on[s]) {
        if (k.lfail[s] != RG_NONE) l = k.lfail[s];
        else if (k.cfail[s] != RG_NONE) l = k.cfail[s];
        else if (k.rfail[s] != RG_NONE) l = val[k.rlast[s] >= 0 ? k.rlast[s] : k.rfirst[s]] - m - n_t;
    }
    fidx[s] = l >= 0 ? l_cidx[l] : INT_MIN;
}

// thread per lookup: lookup_read (the completion :index of the read at its position, JTB_SW_AFTER after the last read,
// JTB_SW_NEVER on a shard not proved with its lookups)
__global__ void lk_lookup_read(RgDev x, TlDev d, TpDev p, LkDev k, const int32_t* __restrict__ rd_cidx,
                               int32_t* __restrict__ lread) {
    const int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (l >= d.n_l) return;
    const int32_t s = d.l_shard[l];
    int32_t v = JTB_SW_NEVER;
    if (lk_ok(k, s)) v = k.lpos[l] < lk_end(p, s) ? rd_cidx[x.ord[k.lpos[l]]] : JTB_SW_AFTER;
    lread[l] = v;
}

// thread per transfer: 1 for a crashed transfer of a proved shard that commits after the last read because a lookup
// returns it
__global__ void lk_after(TpDev p, LkDev k, uint8_t* __restrict__ after) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t];
    after[t] = lk_ok(k, s) && p.t_fate[t] != JTB_T_OK && k.G[t] == lk_end(p, s);
}

// ---- host ---------------------------------------------------------------------------------------------------------

// the per-shard lookup fields K17 adds to K16's
struct LkOut {
    std::vector<int32_t> cause, fail_index;
    std::vector<int64_t> placed;
    std::vector<int32_t> lread;   // per :ok lookup
};

// K17's pass over K16's results (run_repairs' Pass): CwPass, then the lookup pass
struct LkPass {
    CwPass cw;
    LkOut* out = nullptr;

    int pre(cudaStream_t st, TpStage& g, std::string& err) { return cw.pre(st, g, err); }

    int post(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, TpStage& g, int32_t max_rounds,
             jtb_cw_shard* shards, std::vector<int32_t>& cr_h, float& ms, std::string& err) {
        const int32_t S = g.S, nT = g.nT, nL = g.nL, m = g.m;
        const int64_t nR = g.nR;
        const TlHost& T = g.T;
        // the class pass runs on the shards K15 leaves so (CwPass::post's condition); K15's owners before it
        std::vector<uint8_t> cls(S, 0);
        for (int32_t s = 0; s < S; ++s) {
            const jtb_cw_shard& o = shards[s];
            cls[s] = g.dev[s] && o.valid == JTB_UNKNOWN &&
                     (o.cause == JTB_CAUSE_UNDECIDED || o.cause == JTB_CAUSE_NO_WITNESS || o.cause == JTB_CAUSE_REAL_TIME);
        }
        CallAllocs& A = g.A;
        int32_t* kowner;
        JTB_OK(A.alloc(&kowner, nT));
        if (nT > 0) JTB_OK(cudaMemcpyAsync(kowner, g.p.owner, (size_t)nT * 4, cudaMemcpyDeviceToDevice, st));
        if (int rc = cw.post(st, ev0, ev1, h, g, max_rounds, shards, cr_h, ms, err)) return rc;
        std::vector<uint8_t> on(S, 0);
        bool any = false;
        for (int32_t s = 0; s < S; ++s)
            any |= (on[s] = g.dev[s] && shards[s].valid == JTB_VALID && T.lk_off[s + 1] > T.lk_off[s]);
        if (!any) return 0;
        if ((int64_t)m + nT + nL > INT_MAX) { err = "more than 2^31-1 reads, transfers and lookups"; return -2; }
        RgDev& x = g.x;
        TpDev& p = g.p;
        TlDev& d = g.d;
        LkDev k;
        k.kowner = kowner;
        const int64_t nE = (int64_t)m + nT + nL;
        const int32_t nH = m + S;
        std::vector<int32_t> rd_cidx(m);
        for (int32_t i = 0; i < m; ++i) rd_cidx[i] = h->index[g.H.r_ev[g.d_of[i]]];
        int32_t *hist, *gmax, *Q, *lperm0, *lperm, *head, *lcnt, *ccum, *oval0, *oval, *skey, *xin, *P;
        LkKey *lkey0, *lkey;
        LkOpKey *okey0, *okey;
        uint8_t *live, *stmp;
        JTB_OK(A.put(&k.on, on, st)); JTB_OK(A.put(&k.cls, cls, st)); JTB_OK(A.put(&k.l_inv, T.l_inv, st));
        JTB_OK(A.alloc(&k.shown, nT)); JTB_OK(A.alloc(&k.G, nT)); JTB_OK(A.alloc(&k.layer, nT));
        JTB_OK(A.alloc(&hist, nH)); JTB_OK(A.alloc(&k.cum, nH)); JTB_OK(A.alloc(&gmax, m)); JTB_OK(A.alloc(&Q, m));
        JTB_OK(A.alloc(&k.lo, nL)); JTB_OK(A.alloc(&k.below, nL)); JTB_OK(A.alloc(&k.bad, nL));
        JTB_OK(A.alloc(&k.lpos, nL)); JTB_OK(A.alloc(&k.la, nL)); JTB_OK(A.alloc(&k.grank, nL));
        JTB_OK(A.alloc(&head, nL)); JTB_OK(A.alloc(&k.gstart, nL)); JTB_OK(A.alloc(&lcnt, nL));
        JTB_OK(A.alloc(&ccum, nL)); JTB_OK(A.alloc(&lkey0, nL)); JTB_OK(A.alloc(&lkey, nL));
        JTB_OK(A.alloc(&lperm0, nL)); JTB_OK(A.alloc(&lperm, nL));
        JTB_OK(A.alloc(&k.lfail, S)); JTB_OK(A.alloc(&k.cfail, S)); JTB_OK(A.alloc(&k.rfail, S));
        JTB_OK(A.alloc(&k.rlast, S)); JTB_OK(A.alloc(&k.rfirst, S)); JTB_OK(A.alloc(&live, S));
        const int32_t *d_rcidx, *d_lcidx;
        int32_t *fidx, *lread;
        uint8_t* after;
        JTB_OK(A.put(&d_rcidx, rd_cidx, st)); JTB_OK(A.put(&d_lcidx, T.l_cidx, st));
        JTB_OK(A.alloc(&fidx, S)); JTB_OK(A.alloc(&lread, nL)); JTB_OK(A.alloc(&after, nT));
        JTB_OK(A.alloc(&okey0, nE)); JTB_OK(A.alloc(&okey, nE)); JTB_OK(A.alloc(&oval0, nE)); JTB_OK(A.alloc(&oval, nE));
        JTB_OK(A.alloc(&skey, nE)); JTB_OK(A.alloc(&xin, nE)); JTB_OK(A.alloc(&P, nE));
        k.Q = Q;
        // cub's temporary storage: the largest of its uses
        size_t stmp_bytes = 0, b = 0;
        auto need = [&](cudaError_t e) {
            stmp_bytes = std::max(stmp_bytes, b);
            return e;
        };
        JTB_OK(need(cub::DeviceScan::InclusiveSum(nullptr, b, hist, k.cum, nH, st)));
        JTB_OK(need(cub::DeviceScan::InclusiveScanByKey(nullptr, b, skey, xin, P, MaxOp{}, nE, cuda::std::equal_to<>{},
                                                        st)));
        JTB_OK(need(cub::DeviceScan::InclusiveScanByKey(nullptr, b, skey, xin, Q, MaxOp{}, m, cuda::std::equal_to<>{},
                                                        st)));
        JTB_OK(need(cub::DeviceRadixSort::SortPairs(nullptr, b, lkey0, lkey, lperm0, lperm, nL, LkKeyDecomposer{}, st)));
        JTB_OK(need(cub::DeviceScan::InclusiveScan(nullptr, b, head, k.gstart, MaxOp{}, nL, st)));
        JTB_OK(need(cub::DeviceScan::InclusiveSum(nullptr, b, lcnt, ccum, nL, st)));
        JTB_OK(need(cub::DeviceRadixSort::SortPairs(nullptr, b, okey0, okey, oval0, oval, nE, LkOpKeyDecomposer{}, st)));
        JTB_OK(A.alloc(&stmp, stmp_bytes));
        auto grid = [](int64_t n, int per) { return (unsigned)std::max<int64_t>(1, (n + per - 1) / per); };
        size_t tb;
        // G, N and Q
        JTB_OK(cudaMemsetAsync(k.shown, 0, (size_t)nT, st));
        JTB_OK(cudaMemsetAsync(hist, 0, (size_t)nH * 4, st));
        JTB_OK(cudaMemsetAsync(gmax, 0x80, (size_t)m * 4, st));   // INT_MIN
        JTB_OK(cudaMemsetAsync(k.layer, 0x7f, (size_t)nT * 4, st));   // RG_NONE
        if (nR > 0) lk_shown<<<grid(nR, 256), 256, 0, st>>>(d, k);
        if (nT > 0) lk_gap<<<grid(nT, 256), 256, 0, st>>>(p, k, hist, gmax);
        tb = stmp_bytes;
        JTB_OK(cub::DeviceScan::InclusiveSum(stmp, tb, hist, k.cum, nH, st));
        {
            SwDev w;
            w.gmax = gmax;
            w.skey = skey;
            w.x = xin;
            sw_scan_in<<<grid(m, 256), 256, 0, st>>>(x, w);
            tb = stmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, skey, xin, Q, MaxOp{}, m, cuda::std::equal_to<>{},
                                                       st));
        }
        // the ranges and the positions
        lk_linit<<<grid(nL, 256), 256, 0, st>>>(d, p, k);
        JTB_OK(cudaMemsetAsync(k.lfail, 0x7f, (size_t)S * 4, st));   // RG_NONE
        JTB_OK(cudaMemsetAsync(k.cfail, 0x7f, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(k.rfail, 0x7f, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(k.rlast, 0xff, (size_t)S * 4, st));
        JTB_OK(cudaMemsetAsync(k.rfirst, 0x7f, (size_t)S * 4, st));
        if (nR > 0) {
            lk_rec<<<grid(nR, 256), 256, 0, st>>>(d, p, k);
            lk_below<<<grid(nR, 256), 256, 0, st>>>(d, k);
        }
        lk_place<<<grid(nL, 256), 256, 0, st>>>(d, p, k, lkey0, lperm0);
        tb = stmp_bytes;
        JTB_OK(cub::DeviceRadixSort::SortPairs(stmp, tb, lkey0, lkey, lperm0, lperm, nL, LkKeyDecomposer{}, st));
        lk_heads<<<grid(nL, 256), 256, 0, st>>>(nL, lkey, lperm, k, head);
        tb = stmp_bytes;
        JTB_OK(cub::DeviceScan::InclusiveScan(stmp, tb, head, k.gstart, MaxOp{}, nL, st));
        // the shards whose lookups all have a place: the chain test
        std::vector<int32_t> lfail_h(S), fidx_h(S);
        JTB_OK(cudaMemcpyAsync(lfail_h.data(), k.lfail, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        std::vector<uint8_t> live_h(S, 0);
        for (int32_t s = 0; s < S; ++s) live_h[s] = on[s] && lfail_h[s] == RG_NONE;
        JTB_OK(cudaMemcpyAsync(live, live_h.data(), (size_t)S, cudaMemcpyHostToDevice, st));
        JTB_OK(cudaMemsetAsync(lcnt, 0, (size_t)nL * 4, st));
        if (nR > 0) lk_layer<<<grid(nR, 256), 256, 0, st>>>(d, k, live);
        if (nT > 0) lk_lcount<<<grid(nT, 256), 256, 0, st>>>(nT, k, lcnt);
        tb = stmp_bytes;
        JTB_OK(cub::DeviceScan::InclusiveSum(stmp, tb, lcnt, ccum, nL, st));
        lk_chain<<<grid(nL, 256), 256, 0, st>>>(d, k, lperm, ccum, live);
        // the merged order and its real-time pass
        lk_ops<<<grid(nE, 256), 256, 0, st>>>(x, d, p, k, live, okey0, oval0);
        tb = stmp_bytes;
        JTB_OK(cub::DeviceRadixSort::SortPairs(stmp, tb, okey0, okey, oval0, oval, nE, LkOpKeyDecomposer{}, st));
        lk_scan_in<<<grid(nE, 256), 256, 0, st>>>(nE, x, d, p, k, okey, oval, skey, xin);
        tb = stmp_bytes;
        JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, tb, skey, xin, P, MaxOp{}, nE, cuda::std::equal_to<>{}, st));
        lk_rt<<<grid(nE, 256), 256, 0, st>>>(nE, x, d, p, k, okey, oval, P);
        lk_rt_lookup<<<grid(nE, 256), 256, 0, st>>>(nE, x, p, d, k, okey, oval);
        lk_fail_index<<<grid(S, 256), 256, 0, st>>>(S, m, nT, k, d_lcidx, oval, fidx);
        lk_lookup_read<<<grid(nL, 256), 256, 0, st>>>(x, d, p, k, d_rcidx, lread);
        if (nT > 0) lk_after<<<grid(nT, 256), 256, 0, st>>>(p, k, after);
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<uint8_t> after_h(nT);
        JTB_OK(cudaMemcpyAsync(fidx_h.data(), fidx, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        if (nL > 0) JTB_OK(cudaMemcpyAsync(out->lread.data(), lread, (size_t)nL * 4, cudaMemcpyDeviceToHost, st));
        if (nT > 0) JTB_OK(cudaMemcpyAsync(after_h.data(), after, (size_t)nT, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        for (int32_t s = 0; s < S; ++s) {
            if (!on[s]) continue;
            jtb_cw_shard& o = shards[s];
            if (fidx_h[s] != INT_MIN) {
                o.valid = JTB_UNKNOWN;
                o.cause = JTB_CAUSE_LOOKUP;
                o.fail_index = fidx_h[s];
                o.transfer_id = -1;
                o.n_committed = o.n_committed_crashed = o.n_after = 0;
                out->cause[s] = JTB_CAUSE_LOOKUP;
                out->fail_index[s] = fidx_h[s];
                continue;
            }
            for (int32_t t = T.t_off[s]; t < T.t_off[s + 1]; ++t)
                if (after_h[t]) cr_h[t] = JTB_SW_AFTER;
            out->placed[s] = T.lk_off[s + 1] - T.lk_off[s];
        }
        return 0;
    }
};

inline int run_lookup_witness(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                              int64_t max_nodes, int32_t max_rounds, int32_t max_repairs, int32_t max_lifts,
                              int32_t flags, int32_t* commit_read, int32_t* lookup_read, jtb_lk_shard* shards,
                              jtb_lk_result* out, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    const int32_t S = std::max(h->n_shards, 0);
    // the :ok lookups of every shard (tl_host_pass's), and the first one's completion :index
    std::vector<int64_t> nl(S, 0);
    std::vector<int32_t> first(S, -1);
    int64_t nL = 0;
    for (int32_t s = 0; s < S; ++s)
        for (int64_t e = h->shard_off[s]; e < h->shard_off[s + 1]; ++e)
            if (h->process[e] >= 0 && h->type[e] == JTB_T_OK && h->f[e] == JTB_F_LOOKUP && h->payload_len[e] >= 0) {
                if (nl[s]++ == 0) first[s] = h->index[e];
                nL++;
            }
    std::vector<jtb_cw_shard> cw(std::max(S, 1));
    jtb_cw_result cr;
    LkOut lo;
    lo.cause.assign(S, 0);
    lo.fail_index.assign(S, -1);
    lo.placed.assign(S, 0);
    lo.lread.assign(nL, JTB_SW_NEVER);
    LkPass pass;
    pass.out = &lo;
    if (int rc = run_repairs(st, ev0, ev1, h, max_nodes, max_rounds, max_repairs, max_lifts, commit_read, cw.data(),
                             &cr, flags, err, pass))
        return rc;
    memset(out, 0, sizeof *out);
    int64_t at = 0;
    for (int32_t s = 0; s < S; ++s) {
        const jtb_cw_shard& c = cw[s];
        jtb_lk_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = c.valid; o.cause = c.cause; o.n_reads = c.n_reads; o.n_transfers = c.n_transfers;
        o.n_committed = c.n_committed; o.n_committed_crashed = c.n_committed_crashed; o.n_after = c.n_after;
        o.nodes = c.nodes; o.rounds = c.rounds; o.fail_index = c.fail_index; o.transfer_id = c.transfer_id;
        o.repairs = c.repairs; o.n_bans = c.n_bans; o.lifts = c.lifts; o.n_lifted = c.n_lifted;
        o.class_cause = c.class_cause; o.class_rounds = c.class_rounds; o.n_handed = c.n_handed;
        o.lookup_cause = lo.cause[s];
        o.lookup_fail_index = lo.fail_index[s];
        o.n_lookups_placed = lo.placed[s];
        // a proved shard without reads has no serial order to place its lookups in
        if (o.valid == JTB_VALID && o.n_reads == 0 && nl[s] > 0) {
            o.valid = JTB_UNKNOWN;
            o.cause = o.lookup_cause = JTB_CAUSE_LOOKUP;
            o.fail_index = o.lookup_fail_index = first[s];
            if (commit_read)
                for (int32_t t = 0; t < o.n_transfers; ++t) commit_read[at + t] = JTB_SW_NEVER;
        }
        at += o.n_transfers;
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
    if (lookup_read && nL > 0) memcpy(lookup_read, lo.lread.data(), (size_t)nL * 4);
    roll_up(out, shards, S, (float)(cr.seconds_kernel * 1e3), t0);
    return 0;
}

}  // namespace jtb
