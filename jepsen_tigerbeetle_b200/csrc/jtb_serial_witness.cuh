// jtb_serial_witness.cuh — K13: the serial-witness check (pick one explanation per read gap from the placed transfers
// and check the serial order it gives) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K13 serial-witness check").  K12 runs unchanged up to its finals
// (tp_stage, tp_finals); a shard K12 calls VALID gets a witness.  Then:
//   - sw_init, a thread per gap: a gap is fixed from the start when its Delta' (Delta minus what K12 placed in it) is
//     zero, or when its shard gets no witness; the unfixed ones are counted;
//   - the witness rounds, Jacobi: sw_gaps, a warp per unfixed gap, is tp_gaps' round >= 1 gather (rg_gather, in-window
//     and unowned, amount <= Delta') and one rx_search; an EXPLAINED search leaves one solution in the warp's W.st /
//     W.idx, which becomes the gap's choice (kept in K12's poss rows), and every chosen transfer takes the smallest
//     choosing gap (atomicMin); a gap the search does not explain fails its shard.  sw_fix, a thread per gap: a gap
//     whose every chosen transfer took it is fixed and owns them; the gaps of a failed shard stop; the unfixed ones are
//     counted into the one word the host reads per round;
//   - the real time: sw_tgap, a thread per transfer, the largest invocation and the smallest completion of every gap's
//     D_g (integer atomics) and D_g's counters into K12's owned matrix, cleared first; sw_scan_in and cub's
//     InclusiveScanByKey (max, keyed by shard) give P_j for every read; sw_rt, a thread per gap, and sw_after, a thread
//     per :ok transfer in no gap, the smallest failure key per shard; sw_rt_id the smallest failing transfer id there;
//   - sw_sum, a warp per gap: D_g's counters against V (a mismatch is an internal error);
//   - sw_commit, a thread per transfer: commit_read.
// The host runs these through run_witness (jtb_witness.cuh) with no repairs and no lifts: after the real time,
// rw_verdict (K14's) turns each shard's failure into its cause and key, and sw_commit runs on the shards it proves.
// The decision, the node counts and the rounds equal the SW_SEARCH CPU test oracle's, shard for shard, and commit_read
// entry for entry.
#pragma once
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/jtb_check.h"
#include "jtb_call.cuh"
#include "jtb_read_explanations.cuh"
#include "jtb_read_gaps.cuh"
#include "jtb_transfer_placement.cuh"

namespace jtb {

constexpr int SW_COUNTERS = 4;   // per shard: committed, committed crashed, after, nodes

struct SwDev {
    int32_t round = 0;
    const uint8_t* sok = nullptr;         // [n_shards] K12 VALID and on the device: the shard gets a witness
    const int32_t* t_okcomp = nullptr;    // [n_t] :ok completion position, INT_MAX unless :ok
    uint8_t* fixed = nullptr;             // [m] the gap needs no more rounds
    int32_t* cmin = nullptr;              // [n_t] this round: the smallest gap that chose the transfer, RG_NONE none
    int32_t* sfail = nullptr;             // [n_shards] the smallest gap a round did not explain, RG_NONE none
    int32_t* sunf = nullptr;              // [n_shards] after the last round: the smallest unfixed gap, RG_NONE none
    int32_t* unfixed = nullptr;           // the gaps left to run
    unsigned long long* cnt = nullptr;    // [n_shards * SW_COUNTERS]
    // real time
    int32_t* gmax = nullptr;              // [m] the largest invocation in D_g, INT_MIN none
    int32_t* gmin = nullptr;              // [m] the smallest :ok completion in D_g, INT_MAX none
    int32_t* skey = nullptr;              // [m] the shard at each position (the scan's key)
    int32_t* x = nullptr;                 // [m] max(iv(r), gmax)
    int32_t* P = nullptr;                 // [m] the point of the read at each position
    unsigned long long* rtkey = nullptr;  // [n_shards] min of position << 1 | (1: read, 0: transfer)
    unsigned long long* rtid = nullptr;   // [n_shards] min of id ^ 2^63 of the failing transfers at rtkey
    unsigned int* bad = nullptr;          // gap counters that do not add up
};

// the shard gets a witness and no round failed it
__device__ __forceinline__ bool sw_live(const SwDev& w, int32_t s) {
    return w.sok[s] && w.sfail[s] == RG_NONE && w.sunf[s] == RG_NONE;
}

// thread per gap
__global__ void sw_init(RgDev d, TpDev p, SwDev w) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.m) return;
    const int32_t u = d.ord[i], s = d.shard[u], K = d.n_keys[s];
    bool zero = true;
    if (w.sok[s]) {
        const int32_t lower = i > 0 && d.shard[d.ord[i - 1]] == s ? d.ord[i - 1] : -1;
        const int64_t* vu = d.V + d.row[u];
        const int64_t* vl = lower >= 0 ? d.V + d.row[lower] : nullptr;
        const int64_t* ow = p.own + d.row[u];
        for (int32_t j = 0; j < K && zero; ++j) zero = vu[j] - (vl ? vl[j] : 0) - ow[j] == 0;
    }
    w.fixed[i] = zero;
    if (!zero) atomicAdd(w.unfixed, 1);
}

// one warp, gap i: gather the candidates `take` admits (with rg_gather's own filters) and run one search; on EXPLAINED
// its first solution goes into the gap's row of K12's poss (pn = chosen) and every chosen transfer takes the smallest
// choosing gap (atomicMin into w.cmin); cap goes to rg_gather
template <class Take, class Cap = RgNoCap>
__device__ __forceinline__ bool sw_solve(const RgDev& d, const TpDev& p, const SwDev& w, RgWarp& G, int lane,
                                         int32_t i, Take take, int64_t& nodes, int32_t& chosen, Cap cap = {}) {
    RxWarp& W = G.x;
    const int32_t u = d.ord[i], s = d.shard[u], K = d.n_keys[s], cp = d.comp[u];
    const int32_t lower = i > 0 && d.shard[d.ord[i - 1]] == s ? d.ord[i - 1] : -1;
    const int32_t ivl = lower >= 0 ? d.inv[lower] : -1;
    bool ok = false;
    if (K <= JTB_RG_MAX_KEYS) {
        const int64_t* vu = d.V + d.row[u];
        const int64_t* vl = lower >= 0 ? d.V + d.row[lower] : nullptr;
        const int64_t* ow = p.own + d.row[u];
        const int32_t* kt = d.keys + d.key_off[s];
        bool neg = false;
        for (int32_t j = lane; j < K; j += 32) {
            const int64_t x = vu[j] - (vl ? vl[j] : 0) - ow[j];
            W.key[j] = kt[j];
            W.d[j] = x;
            neg |= x < 0;
        }
        neg = __any_sync(0xffffffffu, neg);
        __syncwarp();
        if (!neg) {
            const int32_t n = rg_gather(d, G, s, K, cp, ivl, lane, take, cap);
            __syncwarp();
            if (n <= JTB_RG_MAX_GATHER) {
                int32_t root_key, kept;
                ok = rx_search(W, K, n, -1, d.max_nodes, lane, nodes, root_key, kept) == RX_EXPLAINED;
                if (ok) {
                    // closed at the root (one node): W.st by candidate over [0, n); else by list position over
                    // [0, kept), the candidate at W.idx
                    const bool root = nodes == 1;
                    const int32_t lim = root ? n : kept;
                    int32_t* ps = p.poss + (int64_t)i * JTB_TP_MAX_GATHER;
                    for (int32_t base = 0; base < lim; base += 32) {
                        const int32_t c = base + lane;
                        const bool in = c < lim && W.st[c] == RX_IN;
                        const unsigned bal = __ballot_sync(0xffffffffu, in);
                        if (in) {
                            const int32_t t = G.ct[root ? c : W.idx[c]];
                            ps[chosen + __popc(bal & ((1u << lane) - 1))] = t;
                            atomicMin(&w.cmin[t], i);
                        }
                        chosen += __popc(bal);
                    }
                }
            }
        }
    }
    return ok;
}

// warp per unfixed gap: the gather of a K12 round >= 1 and one search; its first solution is the gap's choice
__global__ void __launch_bounds__(RG_WARPS * 32) sw_gaps(RgDev d, TpDev p, SwDev w) {
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
    }, nodes, chosen);
    if (lane != 0) return;
    atomicAdd(&w.cnt[(int64_t)s * SW_COUNTERS + 3], (unsigned long long)nodes);
    atomicMax(&p.srounds[s], w.round + 1);
    p.pn[i] = chosen;
    if (!ok) atomicMin(&w.sfail[s], i);
}

// thread per gap: fix the gaps no smaller gap of the round competes with; stop the gaps of a failed shard
__global__ void sw_fix(int32_t m, RgDev d, TpDev p, SwDev w) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= m || w.fixed[i]) return;
    if (w.sfail[d.shard[d.ord[i]]] != RG_NONE) { w.fixed[i] = 1; return; }
    const int32_t n = p.pn[i];
    const int32_t* ps = p.poss + i * JTB_TP_MAX_GATHER;
    bool fix = true;
    for (int32_t c = 0; c < n && fix; ++c) fix = w.cmin[ps[c]] == i;
    if (!fix) { atomicAdd(w.unfixed, 1); return; }
    for (int32_t c = 0; c < n; ++c) p.owner[ps[c]] = (int32_t)i;
    w.fixed[i] = 1;
}

// thread per gap, after the last round: the smallest unfixed gap of every shard
__global__ void sw_unfixed(int32_t m, RgDev d, SwDev w) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < m && !w.fixed[i]) atomicMin(&w.sunf[d.shard[d.ord[i]]], (int32_t)i);
}

// thread per transfer: D_g's invocation max, completion min and counters; the counts
__global__ void sw_tgap(RgDev d, TpDev p, SwDev w) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t], g = p.owner[t];
    if (!sw_live(w, s) || g == RG_NONE) return;
    atomicMax(&w.gmax[g], p.t_inv[t]);
    atomicMin(&w.gmin[g], w.t_okcomp[t]);
    unsigned long long* c = w.cnt + (int64_t)s * SW_COUNTERS;
    atomicAdd(&c[0], 1ull);
    if (p.t_fate[t] != JTB_T_OK) atomicAdd(&c[1], 1ull);
    const int64_t a = d.t_rec[3 * t + 2];
    int64_t* ow = p.own + d.row[d.ord[g]];
    if (p.jd[t] >= 0) atomicAdd((unsigned long long*)&ow[p.jd[t]], (unsigned long long)a);
    if (p.jc[t] >= 0) atomicAdd((unsigned long long*)&ow[p.jc[t]], (unsigned long long)a);
}

// thread per position: the scan's key and input
__global__ void sw_scan_in(RgDev d, SwDev w) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.m) return;
    const int32_t u = d.ord[i];
    w.skey[i] = d.shard[u];
    w.x[i] = max(d.inv[u], w.gmax[i]);
}

// thread per gap: P_j < cp(r_j), and P_{j-1} < cp(t) for t in D_g of a gap with a lower read
__global__ void sw_rt(RgDev d, TpDev p, SwDev w) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.m) return;
    const int32_t u = d.ord[i], s = d.shard[u];
    if (!sw_live(w, s)) return;
    if (i > p.rs_off[s] && w.gmin[i] <= w.P[i - 1]) atomicMin(&w.rtkey[s], (unsigned long long)i << 1);
    if (w.P[i] >= d.comp[u]) atomicMin(&w.rtkey[s], (unsigned long long)i << 1 | 1);
}

// the failure key of transfer t in a live shard, ~0 none
__device__ __forceinline__ unsigned long long sw_tkey(const TpDev& p, const SwDev& w, int64_t t,
                                                      int32_t s) {
    const int32_t g = p.owner[t], cp = w.t_okcomp[t];
    if (g != RG_NONE) return g > p.rs_off[s] && cp <= w.P[g - 1] ? (unsigned long long)g << 1 : ~0ull;
    const int32_t end = p.rs_off[s + 1];
    if (p.t_fate[t] == JTB_T_OK && (p.flag[t] & TP_WIN) && cp <= w.P[end - 1]) return (unsigned long long)end << 1;
    return ~0ull;
}

// thread per transfer: the :ok transfers in no gap commit after the last read
__global__ void sw_after(RgDev d, TpDev p, SwDev w) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t];
    if (!sw_live(w, s) || p.owner[t] != RG_NONE || p.t_fate[t] != JTB_T_OK || !(p.flag[t] & TP_WIN)) return;
    atomicAdd(&w.cnt[(int64_t)s * SW_COUNTERS + 2], 1ull);
    const unsigned long long k = sw_tkey(p, w, t, s);
    if (k != ~0ull) atomicMin(&w.rtkey[s], k);
}

// thread per transfer: the smallest id among the failing transfers at the shard's failure key
__global__ void sw_rt_id(RgDev d, TpDev p, SwDev w) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t];
    if (!sw_live(w, s) || w.rtkey[s] == ~0ull || (w.rtkey[s] & 1)) return;
    if (sw_tkey(p, w, t, s) == w.rtkey[s]) atomicMin(&w.rtid[s], (unsigned long long)d.t_id[t] ^ 0x8000000000000000ull);
}

// warp per gap: D_g's counters against the change V(r_{g+1}) - V(r_g)
__global__ void sw_sum(RgDev d, TpDev p, SwDev w) {
    const int64_t wi = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (wi >= d.m) return;
    const int32_t i = (int32_t)wi, u = d.ord[i], s = d.shard[u], K = d.n_keys[s];
    if (!sw_live(w, s)) return;
    const int32_t lower = i > 0 && d.shard[d.ord[i - 1]] == s ? d.ord[i - 1] : -1;
    const int64_t* vu = d.V + d.row[u];
    const int64_t* vl = lower >= 0 ? d.V + d.row[lower] : nullptr;
    const int64_t* ow = p.own + d.row[u];
    for (int32_t j = lane; j < K; j += 32)
        if (ow[j] != vu[j] - (vl ? vl[j] : 0)) atomicAdd(w.bad, 1u);
}

// thread per transfer: commit_read of the shards on the device (the host fills the others and the failed ones)
__global__ void sw_commit(RgDev d, TpDev p, SwDev w, const int32_t* __restrict__ rd_cidx, int32_t* __restrict__ cr) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t], g = p.owner[t];
    int32_t v = JTB_SW_NEVER;
    if (sw_live(w, s)) {
        if (g != RG_NONE) v = rd_cidx[d.ord[g]];
        else if (p.t_fate[t] == JTB_T_OK) v = (p.flag[t] & TP_WIN) ? JTB_SW_AFTER : JTB_SW_FREE;
    }
    cr[t] = v;
}

// ---- host ---------------------------------------------------------------------------------------------------------

// the completion :index of the read at each sorted position
inline std::vector<int32_t> sw_rd_cidx(const jtb_history* h, const TpStage& g) {
    std::vector<int32_t> c(g.m);
    for (int32_t i = 0; i < g.m; ++i) c[i] = h->index[g.H.r_ev[g.d_of[i]]];
    return c;
}

// the witness state of the stage's gaps, transfers and shards, on the shards sok marks; failures, counters and the
// unfixed count reset
inline int sw_alloc(cudaStream_t st, TpStage& g, const std::vector<uint8_t>& sok, SwDev& w, std::string& err) {
    CallAllocs& A = g.A;
    const int32_t S = g.S, nT = g.nT, m = g.m;
    w.t_okcomp = g.d.t_okcomp;
    JTB_OK(A.put(&w.sok, sok, st));
    JTB_OK(A.alloc(&w.fixed, m)); JTB_OK(A.alloc(&w.cmin, nT)); JTB_OK(A.alloc(&w.sfail, S));
    JTB_OK(A.alloc(&w.sunf, S)); JTB_OK(A.alloc(&w.unfixed, 1)); JTB_OK(A.alloc(&w.cnt, (size_t)S * SW_COUNTERS));
    JTB_OK(A.alloc(&w.gmax, m)); JTB_OK(A.alloc(&w.gmin, m)); JTB_OK(A.alloc(&w.skey, m));
    JTB_OK(A.alloc(&w.x, m)); JTB_OK(A.alloc(&w.P, m)); JTB_OK(A.alloc(&w.rtkey, S)); JTB_OK(A.alloc(&w.rtid, S));
    JTB_OK(A.alloc(&w.bad, 1));
    JTB_OK(cudaMemsetAsync(w.sfail, 0x7f, (size_t)S * 4, st));   // RG_NONE
    JTB_OK(cudaMemsetAsync(w.sunf, 0x7f, (size_t)S * 4, st));
    JTB_OK(cudaMemsetAsync(w.cnt, 0, (size_t)S * SW_COUNTERS * 8, st));
    JTB_OK(cudaMemsetAsync(w.unfixed, 0, 4, st));
    return 0;
}

// the real time and the counters of the witness in p.owner: sw_tgap over owned counters cleared first, the max-scan
// (cub's temporary storage stmp), sw_rt, sw_sum and sw_after; sw_rt_id and sw_commit are the caller's
inline int sw_real_time(cudaStream_t st, TpStage& g, const SwDev& w, uint8_t* stmp, size_t stmp_bytes,
                        std::string& err) {
    const int32_t S = g.S, nT = g.nT, m = g.m;
    auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };
    JTB_OK(cudaMemsetAsync(w.gmax, 0x80, (size_t)m * 4, st));   // INT_MIN
    JTB_OK(cudaMemsetAsync(w.gmin, 0x7f, (size_t)m * 4, st));   // > every position
    JTB_OK(cudaMemsetAsync(w.rtkey, 0xff, (size_t)S * 8, st));
    JTB_OK(cudaMemsetAsync(w.rtid, 0xff, (size_t)S * 8, st));
    JTB_OK(cudaMemsetAsync(w.bad, 0, 4, st));
    JTB_OK(cudaMemsetAsync(g.own, 0, (size_t)g.cells * 8, st));
    if (nT > 0) sw_tgap<<<grid(nT, 256), 256, 0, st>>>(g.x, g.p, w);
    sw_scan_in<<<grid(m, 256), 256, 0, st>>>(g.x, w);
    JTB_OK(cub::DeviceScan::InclusiveScanByKey(stmp, stmp_bytes, w.skey, w.x, w.P, MaxOp{}, m, cuda::std::equal_to<>{},
                                               st));
    sw_rt<<<grid(m, 256), 256, 0, st>>>(g.x, g.p, w);
    sw_sum<<<grid((int64_t)m * 32, 256), 256, 0, st>>>(g.x, g.p, w);
    if (nT > 0) sw_after<<<grid(nT, 256), 256, 0, st>>>(g.x, g.p, w);
    return 0;
}

}  // namespace jtb
