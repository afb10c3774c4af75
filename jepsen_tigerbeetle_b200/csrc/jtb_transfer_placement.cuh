// jtb_transfer_placement.cuh — K12: the transfer-placement check (carry the transfers each read gap locates into the
// other gaps, to a fixpoint) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K12 transfer-placement check").  The reads, their order, the gaps, the
// transfers, M(t) and A(t) are K11's, with K11's host passes and first kernels unchanged.  Then:
//   - tp_pos, two cub scans and tp_window, a thread per transfer: the window [lo, hi] from one binary search over the
//     shard's reads in completion order (prefix maximum of their positions) and one over its reads by invocation
//     (suffix minimum of their positions), and the columns of its two keys;
//   - the rounds, Jacobi: tp_gaps, a warp per gap to run (every gap in rounds 0 and 1, the dirtied ones after), is
//     rg_gaps with Delta' = Delta - the owned contributions, the in-window, unowned gather from round 1 on (the same
//     rg_gather), the root pruning's possible candidates kept per gap, and the latch; tp_possible, a warp per gap,
//     the smallest and largest possible gap of every must transfer; a cub sum of the incomplete gaps; tp_owner, a
//     thread per transfer, owner, DOUBLE, PLACE and LOST, the owned contributions (integer atomics into a matrix shaped
//     like V) and the difference array of the dirtied windows, summed by cub before the next round; the host reads one
//     changed-flag word per round;
//   - tp_gap_final, tp_transfer_final and tp_witness_id: the counts, the verdict and the witness.
// The host side is two stages: tp_stage (the host passes, the first kernels, the windows and the rounds) and tp_finals;
// the serial-witness check (jtb_serial_witness.cuh) runs both and then its own kernels on the stage's device state.
// The decision, the caps, the node counts and the rounds equal the TP_SEARCH CPU test oracle's, gap for gap.
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
#include "jtb_monotonic.cuh"
#include "jtb_read_explanations.cuh"
#include "jtb_read_gaps.cuh"
#include "jtb_transfer_lookups.cuh"

namespace jtb {

static_assert(JTB_TP_MAX_GATHER == JTB_RG_MAX_GATHER && JTB_TP_KEY == JTB_RG_KEY && JTB_TP_JOINT == JTB_RG_JOINT &&
                  JTB_TP_DOUBLE == JTB_RG_DOUBLE, "K12's round 0 is K11");

constexpr int TP_COUNTERS = 8;   // per shard: explained, undecided, KEY, JOINT, DOUBLE, LOST, placed, nodes
constexpr uint8_t TP_WIN = 1, TP_MUST = 2;

struct TpDev {
    int32_t round = 0;
    int32_t n_t = 0;
    const int32_t* rs_off = nullptr;      // [n_shards + 1] the shard's device reads (and sorted positions)
    const int32_t* pos = nullptr;         // [m] sorted position of each device read
    // per transfer
    const int32_t* t_shard = nullptr;
    const int32_t* t_fate = nullptr;
    const int32_t* t_inv = nullptr;
    int32_t* lo = nullptr;
    int32_t* hi = nullptr;
    int32_t* jd = nullptr;
    int32_t* jc = nullptr;
    uint8_t* flag = nullptr;              // TP_WIN | TP_MUST
    int32_t* owner = nullptr;             // gap, RG_NONE none
    int32_t* pmin = nullptr;              // this round: the smallest / largest possible gap in the window
    int32_t* pmax = nullptr;
    int32_t* dround = nullptr;            // DOUBLE: the round, -1 none, and the two gaps
    int32_t* dg1 = nullptr;
    int32_t* dg2 = nullptr;
    int32_t* lround = nullptr;            // LOST: the round, -1 none
    // per gap (sorted position)
    const int32_t* dirty = nullptr;       // from round 2 on: > 0 = run
    int64_t* own = nullptr;               // shaped like V: the owned contributions by the upper read's row
    int8_t* lcode = nullptr;              // latched KEY / JOINT, 0 none
    int32_t* lround_g = nullptr;
    int32_t* inc = nullptr;               // 1: the gather passed the cap or the shard has too many keys
    const int32_t* incsum = nullptr;      // inclusive sum of inc
    int32_t* pn = nullptr;                // gathered candidates kept in poss
    int32_t* poss = nullptr;              // [m * JTB_TP_MAX_GATHER] the transfer, -1 when the root pruned it out
    int32_t* dd = nullptr;                // [m + 1] difference array of the dirtied windows
    unsigned int* changed = nullptr;
    int32_t* srounds = nullptr;           // [n_shards]
};

struct MaxOp {
    __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return max(a, b); }
};
struct MinOp {
    __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return min(a, b); }
};

// thread per sorted position
__global__ void tp_pos(int32_t m, const int32_t* __restrict__ ord, int32_t* __restrict__ pos) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < m) pos[ord[i]] = (int32_t)i;
}

// thread per k: the positions of the reads by invocation, reversed for the suffix minimum
__global__ void tp_ivpos(int32_t m, const int32_t* __restrict__ ivperm, const int32_t* __restrict__ pos,
                         int32_t* __restrict__ rev) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k < m) rev[m - 1 - k] = pos[ivperm[k]];
}

// thread per transfer: window, must, key columns
__global__ void tp_window(RgDev d, TpDev p, const int32_t* __restrict__ cmax, const int32_t* __restrict__ ivs,
                          const int32_t* __restrict__ srev) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t], r0 = p.rs_off[s], r1 = p.rs_off[s + 1];
    const int32_t* q = d.t_rec + 3 * t;
    int32_t cd = -1, cc = -1;
    uint8_t f = 0;
    if (r1 > r0) {
        const int32_t* kt = d.keys + d.key_off[s];
        const int32_t K = d.n_keys[s];
        auto col = [&](int64_t key) {
            int32_t a = 0, b = K;
            while (a < b) {
                const int32_t c = (a + b) >> 1;
                if (kt[c] < key) a = c + 1; else b = c;
            }
            return a < K && kt[a] == key ? a : -1;
        };
        cd = col(2 * (int64_t)q[0]);
        cc = col(2 * (int64_t)q[1] + 1);
        if (p.t_fate[t] != JTB_T_FAIL && q[2] > 0 && (cd >= 0 || cc >= 0)) {
            f = TP_WIN;
            const int32_t c = rx_lower(d.comp, r0, r1, max(p.t_inv[t], d.t_A[t]));
            p.lo[t] = c > r0 ? cmax[c - 1] + 1 : r0;
            const int32_t M = d.t_M[t];
            const int32_t k = M == INT_MAX ? r1 : rx_lower(ivs, r0, r1, M + 1);
            if (k < r1) f |= TP_MUST;
            p.hi[t] = k < r1 ? srev[d.m - 1 - k] : r1 - 1;
        }
    }
    p.flag[t] = f;
    p.jd[t] = cd;
    p.jc[t] = cc;
}

// warp per gap to run in this round
__global__ void __launch_bounds__(RG_WARPS * 32) tp_gaps(RgDev d, TpDev p) {
    __shared__ RgWarp smem[RG_WARPS];
    const int lane = threadIdx.x & 31;
    RgWarp& G = smem[threadIdx.x >> 5];
    RxWarp& W = G.x;
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (w >= d.m || (p.round >= 2 && p.dirty[w] <= 0)) return;
    const int32_t i = (int32_t)w, u = d.ord[i], s = d.shard[u], K = d.n_keys[s], cp = d.comp[u];
    const int32_t lower = i > 0 && d.shard[d.ord[i - 1]] == s ? d.ord[i - 1] : -1;
    const int32_t ivl = lower >= 0 ? d.inv[lower] : -1;
    const int32_t round = p.round;
    int8_t code = RX_UNDECIDED;
    int64_t nodes = 0, delta = 0;
    int32_t gkey = -1, kept = 0, n = 0, inc = 1;
    if (K <= JTB_RG_MAX_KEYS) {
        inc = 0;
        const int64_t* vu = d.V + d.row[u];
        const int64_t* vl = lower >= 0 ? d.V + d.row[lower] : nullptr;
        const int64_t* ow = p.own + d.row[u];
        const int32_t* kt = d.keys + d.key_off[s];
        int32_t neg = INT_MAX;
        bool nz = false;
        for (int32_t j = lane; j < K; j += 32) {
            const int64_t x = vu[j] - (vl ? vl[j] : 0) - ow[j];
            W.key[j] = kt[j];
            W.d[j] = x;
            if (x < 0) neg = min(neg, j);
            nz |= x != 0;
        }
        neg = rx_warp_min(neg);
        nz = __any_sync(0xffffffffu, nz);
        __syncwarp();
        if (neg != INT_MAX) {
            code = JTB_TP_KEY;
            gkey = W.key[neg];
            delta = W.d[neg];
        } else if (!nz) {
            code = RX_EXPLAINED;
        } else {
            n = rg_gather(d, G, s, K, cp, ivl, lane, [&](int32_t t) {
                return round == 0 || ((p.flag[t] & TP_WIN) && p.lo[t] <= i && i <= p.hi[t] && p.owner[t] == RG_NONE);
            });
            __syncwarp();
            if (n > JTB_RG_MAX_GATHER) {
                inc = 1;
                n = 0;
            } else {
                for (int32_t c = lane; c < n; c += 32) {
                    W.idx[c] = (uint8_t)c;
                    W.st[c] = RX_UND;
                }
                __syncwarp();
                int32_t bad;
                const bool ok = rx_prune(W, K, n, -1, lane, bad);
                int32_t* ps = p.poss + (int64_t)i * JTB_TP_MAX_GATHER;
                for (int32_t c = lane; c < n; c += 32) {
                    ps[c] = W.st[c] != RX_OUT ? G.ct[c] : -1;
                    if (!ok || W.st[c] != RX_IN) continue;
                    const int32_t t = G.ct[c], old = atomicMin(&d.f1[t], i);
                    if (old != RG_NONE) atomicMin(&d.f2[t], max(old, i));
                }
                __syncwarp();
                int32_t root_key;
                code = (int8_t)rx_search(W, K, n, -1, d.max_nodes, lane, nodes, root_key, kept);
                if (code == JTB_TP_JOINT) {
                    gkey = root_key;
                    for (int32_t k = 0; k < K; ++k) {
                        int32_t rk, kp;
                        if (rx_search(W, K, n, k, d.max_nodes, lane, nodes, rk, kp) == JTB_TP_JOINT) {
                            code = JTB_TP_KEY;
                            gkey = W.key[k];
                            delta = W.d[k];
                            break;
                        }
                    }
                }
            }
        }
    }
    if (lane != 0) return;
    atomicAdd(&d.cnt[(int64_t)s * TP_COUNTERS + 7], (unsigned long long)nodes);
    atomicMax(&p.srounds[s], round + 1);
    d.gkept[i] = kept;
    d.code[i] = code;
    p.pn[i] = n;
    p.inc[i] = inc;
    if ((code == JTB_TP_KEY || code == JTB_TP_JOINT) && p.lcode[i] == 0) {
        p.lcode[i] = code;
        p.lround_g[i] = round;
        d.gkey[i] = gkey;
        d.gdelta[i] = delta;
    }
}

// warp per gap: the smallest and the largest gap where each must transfer is still possible
__global__ void tp_possible(int32_t m, TpDev p) {
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= m) return;
    const int32_t i = (int32_t)w, n = p.pn[i];
    const int32_t* ps = p.poss + (int64_t)i * JTB_TP_MAX_GATHER;
    for (int32_t c = lane; c < n; c += 32) {
        const int32_t t = ps[c];
        if (t < 0 || !(p.flag[t] & TP_MUST) || i < p.lo[t] || i > p.hi[t]) continue;
        atomicMin(&p.pmin[t], i);
        atomicMax(&p.pmax[t], i);
    }
}

// thread per transfer: DOUBLE, owner by forcing, PLACE, LOST
__global__ void tp_owner(RgDev d, TpDev p) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const uint8_t f = p.flag[t];
    if (!(f & TP_WIN) || p.owner[t] != RG_NONE || p.dround[t] >= 0 || p.lround[t] >= 0) return;
    const int32_t lo = p.lo[t], hi = p.hi[t];
    int32_t g = -1;
    if (d.f2[t] != RG_NONE) {
        p.dround[t] = p.round;
        p.dg1[t] = d.f1[t];
        p.dg2[t] = d.f2[t];
        return;
    }
    if (d.f1[t] != RG_NONE) {
        g = d.f1[t];
    } else if ((f & TP_MUST) && (lo > hi || p.incsum[hi] - (lo > 0 ? p.incsum[lo - 1] : 0) == 0)) {
        if (p.pmin[t] == RG_NONE) p.lround[t] = p.round;
        else if (p.pmin[t] == p.pmax[t]) g = p.pmin[t];
    }
    if (g < 0) return;
    p.owner[t] = g;
    *p.changed = 1u;
    const int64_t a = d.t_rec[3 * t + 2];
    int64_t* ow = p.own + d.row[d.ord[g]];
    if (p.jd[t] >= 0) atomicAdd((unsigned long long*)&ow[p.jd[t]], (unsigned long long)a);
    if (p.jc[t] >= 0) atomicAdd((unsigned long long*)&ow[p.jc[t]], (unsigned long long)a);
    if (lo <= hi) {
        atomicAdd(&p.dd[lo], 1);
        atomicAdd(&p.dd[hi + 1], -1);
    }
}

// thread per gap: the counts by the latched or last code, the gaps' witness keys
__global__ void tp_gap_final(RgDev d, TpDev p) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.m) return;
    const int32_t s = d.shard[d.ord[i]];
    unsigned long long* c = d.cnt + (int64_t)s * TP_COUNTERS;
    if (p.lcode[i]) {
        atomicAdd(&c[1 + p.lcode[i]], 1ull);
        atomicMin(&d.wkey[s], (unsigned long long)i << 3 | (unsigned)p.lcode[i]);
    } else {
        atomicAdd(&c[d.code[i] == RX_EXPLAINED ? 0 : 1], 1ull);
    }
}

__device__ __forceinline__ unsigned long long tp_tkey(const TpDev& p, int64_t t) {
    if (p.dround[t] >= 0) return (unsigned long long)p.dg2[t] << 3 | JTB_TP_DOUBLE;
    if (p.lround[t] >= 0) return (unsigned long long)p.hi[t] << 3 | JTB_TP_LOST;
    return ~0ull;
}

// thread per transfer: placed, DOUBLE and LOST counts, the transfers' witness keys
__global__ void tp_transfer_final(RgDev d, TpDev p) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const int32_t s = p.t_shard[t];
    unsigned long long* c = d.cnt + (int64_t)s * TP_COUNTERS;
    if (p.owner[t] != RG_NONE) atomicAdd(&c[6], 1ull);
    const unsigned long long k = tp_tkey(p, t);
    if (k == ~0ull) return;
    atomicAdd(&c[(k & 7) == JTB_TP_DOUBLE ? 4 : 5], 1ull);
    atomicMin(&d.wkey[s], k);
}

// thread per transfer: the smallest id among the transfers at their shard's witness
__global__ void tp_witness_id(RgDev d, TpDev p) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= p.n_t) return;
    const unsigned long long k = tp_tkey(p, t);
    if (k != ~0ull && k == d.wkey[p.t_shard[t]])
        atomicMin(&d.wtid[p.t_shard[t]], (unsigned long long)d.t_id[t] ^ 0x8000000000000000ull);
}

// ---- host ---------------------------------------------------------------------------------------------------------

// What K12's stage leaves for the finals of the call that ran it: K7's, K9's and K11's host passes and device reads,
// and the device state at the end of the rounds.
struct TpStage {
    MonoHost H;
    TlHost T;
    int32_t S = 0, nT = 0, nL = 0, m = 0;
    int64_t nR = 0, slots = 0, cells = 0;
    std::vector<char> dev;                // per shard: it has reads and none is partial (its gaps run on the device)
    std::vector<int32_t> d_of, shard_v, inv_v, comp_v, rs_off;
    CallAllocs A;
    TlDev d;
    RgDev x;
    TpDev p;
    int64_t* own = nullptr;
    int32_t* tM = nullptr;
    unsigned long long *cnt = nullptr, *wkey = nullptr, *wtid = nullptr;
    uint8_t* tmp = nullptr;               // cub's temporary storage
    size_t tmp_bytes = 0;
};

// K12 up to its finals: the input checks, the host passes, K7's, K9's and K10's first kernels, the windows and the
// rounds.  With device reads (g.m > 0), ev0 is recorded before the first kernel.
inline int tp_stage(cudaStream_t st, cudaEvent_t ev0, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                    int32_t flags, TpStage& g, std::string& err) {
    if (flags != 0) { err = "flags must be 0 (reserved)"; return -2; }
    if (int rc = check_history(h, false, err)) return rc;
    if (max_nodes <= 0) max_nodes = JTB_TP_DEFAULT_MAX_NODES;
    if (max_rounds <= 0) max_rounds = JTB_TP_DEFAULT_MAX_ROUNDS;
    const int32_t S = g.S = h->n_shards;
    MonoHost& H = g.H;
    if (int rc = mono_host_pass(h, H, err)) return rc;
    TlHost& T = g.T;
    if (int rc = tl_host_pass(h, T, err)) return rc;
    if (T.t_id.size() > (size_t)1 << 30) { err = "more than 2^30 transfers"; return -2; }
    const int32_t nT = g.nT = (int32_t)T.t_id.size(), nL = g.nL = (int32_t)T.l_shard.size();
    const int64_t nR = g.nR = T.rec_base.back(), slots = g.slots = (int64_t)H.keys.size();
    g.dev.assign(S, 0);
    for (int32_t s = 0; s < S; ++s) g.dev[s] = H.n_reads[s] > 0 && H.min_trip[s] >= H.n_keys[s];
    // K11's device reads and sweep structures
    std::vector<int32_t>&d_of = g.d_of, &shard_v = g.shard_v, &inv_v = g.inv_v, &comp_v = g.comp_v, &rs_off = g.rs_off;
    rs_off.assign(S + 1, 0);
    std::vector<int64_t> poff_v, row_v;
    int64_t& cells = g.cells;
    for (int32_t r = 0; r < (int32_t)H.r_shard.size(); ++r) {
        const int32_t s = H.r_shard[r];
        if (!g.dev[s]) continue;
        d_of.push_back(r);
        shard_v.push_back(s);
        inv_v.push_back(H.r_inv[r]);
        comp_v.push_back(H.r_comp[r]);
        poff_v.push_back(H.r_poff[r]);
        row_v.push_back(cells);
        cells += H.n_keys[s];
        rs_off[s + 1]++;
    }
    for (int32_t s = 0; s < S; ++s) rs_off[s + 1] += rs_off[s];
    const int32_t m = g.m = (int32_t)d_of.size();
    if (m == 0) return 0;
    // the device reads of every shard by invocation (stable over completion order)
    std::vector<int32_t> ivperm(m), ivs(m);
    for (int32_t r = 0; r < m; ++r) ivperm[r] = r;
    std::stable_sort(ivperm.begin(), ivperm.end(), [&](int32_t a, int32_t b) {
        return shard_v[a] != shard_v[b] ? shard_v[a] < shard_v[b] : inv_v[a] < inv_v[b];
    });
    for (int32_t k = 0; k < m; ++k) ivs[k] = inv_v[ivperm[k]];
    std::vector<int32_t> ok_t, ok_inv, ok_pmax, ok_off(S + 1, 0), cr_anchor(nT, -1), cr_off(slots + 1, 0);
    for (int32_t s = 0; s < S; ++s) {
        const int32_t* kt = H.keys.data() + H.key_off[s];
        const int32_t K = H.n_keys[s];
        auto col = [&](int64_t key) {
            const int32_t* p = std::lower_bound(kt, kt + K, key, [](int32_t a, int64_t b) { return a < b; });
            return p < kt + K && *p == key ? (int32_t)(p - kt) : -1;
        };
        int32_t run = INT_MIN;
        for (int32_t t = T.t_off[s]; t < T.t_off[s + 1]; ++t) {
            if (T.t_fate[t] == JTB_T_OK) {
                run = std::max(run, T.t_okcomp[t]);
                ok_t.push_back(t);
                ok_inv.push_back(T.t_inv[t]);
                ok_pmax.push_back(run);
            } else if (T.t_fate[t] != JTB_T_FAIL && T.t_rec[3 * (size_t)t + 2] > 0) {
                const int32_t cd = col(2 * (int64_t)T.t_rec[3 * (size_t)t]);
                const int32_t a = cd >= 0 ? cd : col(2 * (int64_t)T.t_rec[3 * (size_t)t + 1] + 1);
                if (a >= 0) cr_off[(cr_anchor[t] = (int32_t)(H.key_off[s] + a)) + 1]++;
            }
        }
        ok_off[s + 1] = (int32_t)ok_t.size();
    }
    for (int64_t k = 0; k < slots; ++k) cr_off[k + 1] += cr_off[k];
    std::vector<int32_t> cr_t(cr_off[slots]), cr_inv(cr_off[slots]), fill(cr_off.begin(), cr_off.end() - 1);
    for (int32_t t = 0; t < nT; ++t)
        if (cr_anchor[t] >= 0) {
            const int32_t j = fill[cr_anchor[t]]++;
            cr_t[j] = t;
            cr_inv[j] = T.t_inv[t];
        }
    CallAllocs& A = g.A;
    int64_t *V, *own;
    if (A.alloc(&V, (size_t)cells) != cudaSuccess || A.alloc(&own, (size_t)cells) != cudaSuccess) {
        err = "cannot allocate the dense value matrices (2 x " + std::to_string((size_t)cells * sizeof(int64_t)) +
              " bytes on the device)";
        return -3;
    }
    TlDev& d = g.d;
    RgDev& x = g.x;
    TpDev& p = g.p;
    d.n_t = nT;
    d.n_l = nL;
    d.n_rec = nR;
    x.m = m;
    x.V = V;
    x.max_nodes = max_nodes;
    p.n_t = nT;
    p.own = g.own = own;
    const int64_t* tid;
    const int64_t* poff;
    TlTKey *tk0, *tk;
    TlRKey *rk0, *rk;
    MonoKey *key0, *key1;
    int32_t *tid0, *tperm, *rv0, *rv, *tM, *tA, *id0, *id1, *pos, *cmax, *srev, *rev, *dirty;
    const int32_t *d_ivperm, *d_ivs;
    uint64_t* mk;
    unsigned long long *cnt, *wkey, *wtid;
    uint8_t* tmp;
    JTB_OK(A.put(&d.payload, h->payload, (size_t)h->n_payload, st));
    JTB_OK(A.put(&poff, poff_v, st)); JTB_OK(A.put(&x.row, row_v, st)); JTB_OK(A.put(&x.shard, shard_v, st));
    JTB_OK(A.put(&x.inv, inv_v, st)); JTB_OK(A.put(&x.comp, comp_v, st));
    JTB_OK(A.put(&d.n_keys, H.n_keys, st)); JTB_OK(A.put(&d.key_off, H.key_off, st)); JTB_OK(A.put(&d.keys, H.keys, st));
    x.n_keys = d.n_keys; x.key_off = d.key_off; x.keys = d.keys;
    JTB_OK(A.put(&d.t_shard, T.t_shard, st)); JTB_OK(A.put(&tid, T.t_id, st)); JTB_OK(A.put(&d.t_rec, T.t_rec, st));
    JTB_OK(A.put(&d.t_inv, T.t_inv, st)); JTB_OK(A.put(&d.t_okcomp, T.t_okcomp, st));
    JTB_OK(A.put(&d.t_fate, T.t_fate, st)); JTB_OK(A.put(&d.t_off, T.t_off, st));
    x.t_rec = d.t_rec; x.t_id = tid;
    JTB_OK(A.put(&d.l_shard, T.l_shard, st)); JTB_OK(A.put(&d.l_comp, T.l_comp, st));
    JTB_OK(A.put(&d.l_poff, T.l_poff, st)); JTB_OK(A.put(&d.rec_base, T.rec_base, st));
    JTB_OK(A.put(&d.ib, T.ib, st)); JTB_OK(A.put(&d.ib_inv, T.ib_inv, st)); JTB_OK(A.put(&d.ib_off, T.ib_off, st));
    JTB_OK(A.put(&x.ok_t, ok_t, st)); JTB_OK(A.put(&x.ok_inv, ok_inv, st)); JTB_OK(A.put(&x.ok_pmax, ok_pmax, st));
    JTB_OK(A.put(&x.ok_off, ok_off, st)); JTB_OK(A.put(&x.cr_t, cr_t, st)); JTB_OK(A.put(&x.cr_inv, cr_inv, st));
    JTB_OK(A.put(&x.cr_off, cr_off, st));
    JTB_OK(A.put(&p.rs_off, rs_off, st)); JTB_OK(A.put(&d_ivperm, ivperm, st)); JTB_OK(A.put(&d_ivs, ivs, st));
    JTB_OK(A.alloc(&key0, m)); JTB_OK(A.alloc(&key1, m)); JTB_OK(A.alloc(&id0, m)); JTB_OK(A.alloc(&id1, m));
    JTB_OK(A.alloc(&tk0, nT)); JTB_OK(A.alloc(&tk, nT)); JTB_OK(A.alloc(&tid0, nT)); JTB_OK(A.alloc(&tperm, nT));
    JTB_OK(A.alloc(&d.rec_slot, nR)); JTB_OK(A.alloc(&rk0, nR)); JTB_OK(A.alloc(&rk, nR));
    JTB_OK(A.alloc(&rv0, nR)); JTB_OK(A.alloc(&rv, nR));
    JTB_OK(A.alloc(&d.mlk, nT)); JTB_OK(A.alloc(&d.mv, nT)); JTB_OK(A.alloc(&d.mfrom, nT)); JTB_OK(A.alloc(&mk, nT));
    JTB_OK(A.alloc(&d.wid, (size_t)nL * 5)); JTB_OK(A.alloc(&d.count, (size_t)S * JTB_TL_KINDS));
    JTB_OK(A.alloc(&tM, nT)); JTB_OK(A.alloc(&tA, nT)); JTB_OK(A.alloc(&x.f1, nT)); JTB_OK(A.alloc(&x.f2, nT));
    JTB_OK(A.alloc(&x.code, m)); JTB_OK(A.alloc(&x.gkey, m)); JTB_OK(A.alloc(&x.gkept, m));
    JTB_OK(A.alloc(&x.gdelta, m));
    JTB_OK(A.alloc(&cnt, (size_t)S * TP_COUNTERS)); JTB_OK(A.alloc(&wkey, S)); JTB_OK(A.alloc(&wtid, S));
    JTB_OK(A.alloc(&pos, m)); JTB_OK(A.alloc(&cmax, m)); JTB_OK(A.alloc(&rev, m)); JTB_OK(A.alloc(&srev, m));
    JTB_OK(A.alloc(&p.lo, nT)); JTB_OK(A.alloc(&p.hi, nT)); JTB_OK(A.alloc(&p.jd, nT)); JTB_OK(A.alloc(&p.jc, nT));
    JTB_OK(A.alloc(&p.flag, nT)); JTB_OK(A.alloc(&p.owner, nT)); JTB_OK(A.alloc(&p.pmin, nT));
    JTB_OK(A.alloc(&p.pmax, nT)); JTB_OK(A.alloc(&p.dround, nT)); JTB_OK(A.alloc(&p.dg1, nT));
    JTB_OK(A.alloc(&p.dg2, nT)); JTB_OK(A.alloc(&p.lround, nT));
    JTB_OK(A.alloc(&p.lcode, m)); JTB_OK(A.alloc(&p.lround_g, m)); JTB_OK(A.alloc(&p.inc, m));
    JTB_OK(A.alloc(&dirty, (size_t)m + 1)); JTB_OK(A.alloc(&p.pn, m)); JTB_OK(A.alloc(&p.dd, (size_t)m + 1));
    JTB_OK(A.alloc(&p.poss, (size_t)m * JTB_TP_MAX_GATHER)); JTB_OK(A.alloc(&p.changed, 1));
    JTB_OK(A.alloc(&p.srounds, S));
    int32_t* incsum;
    JTB_OK(A.alloc(&incsum, m));
    d.tkey = tk; d.tperm = tperm; d.rkey = rk; d.rval = rv;
    x.ord = id1; x.t_M = tM; x.t_A = tA; x.cnt = cnt; x.wkey = wkey; x.wtid = wtid;
    p.pos = pos; p.t_shard = d.t_shard; p.t_fate = d.t_fate; p.t_inv = d.t_inv; p.dirty = dirty;
    p.incsum = incsum;
    g.tM = tM; g.cnt = cnt; g.wkey = wkey; g.wtid = wtid;
    size_t tmp_m = 0, tmp_t = 0, tmp_r = 0, tmp_s = 0, tmp_s2 = 0, tmp_s3 = 0;
    JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_m, key0, key1, id0, id1, m, MonoKeyDecomposer{}, st));
    if (nT > 0)
        JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_t, tk0, tk, tid0, tperm, nT, TlTKeyDecomposer{}, st));
    if (nR > 0)
        JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_r, rk0, rk, rv0, rv, (int)nR, TlRKeyDecomposer{}, st));
    JTB_OK(cub::DeviceScan::InclusiveScan(nullptr, tmp_s, pos, cmax, MaxOp{}, m, st));
    JTB_OK(cub::DeviceScan::InclusiveScan(nullptr, tmp_s2, rev, srev, MinOp{}, m, st));
    JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, tmp_s3, p.dd, dirty, m + 1, st));
    const size_t tmp_bytes = g.tmp_bytes = std::max({tmp_m, tmp_t, tmp_r, tmp_s, tmp_s2, tmp_s3});
    JTB_OK(A.alloc(&tmp, tmp_bytes));
    g.tmp = tmp;
    auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };

    JTB_OK(cudaEventRecord(ev0, st));
    JTB_OK(cudaMemsetAsync(d.mlk, 0x7f, (size_t)nT * 4, st));
    JTB_OK(cudaMemsetAsync(d.wid, 0xff, (size_t)nL * 40, st));
    JTB_OK(cudaMemsetAsync(d.count, 0, (size_t)S * JTB_TL_KINDS * 8, st));
    JTB_OK(cudaMemsetAsync(cnt, 0, (size_t)S * TP_COUNTERS * 8, st));
    JTB_OK(cudaMemsetAsync(wkey, 0xff, (size_t)S * 8, st));
    JTB_OK(cudaMemsetAsync(wtid, 0xff, (size_t)S * 8, st));
    JTB_OK(cudaMemsetAsync(own, 0, (size_t)cells * 8, st));
    JTB_OK(cudaMemsetAsync(p.owner, 0x7f, (size_t)nT * 4, st));   // RG_NONE
    JTB_OK(cudaMemsetAsync(p.dround, 0xff, (size_t)nT * 4, st));
    JTB_OK(cudaMemsetAsync(p.lround, 0xff, (size_t)nT * 4, st));
    JTB_OK(cudaMemsetAsync(p.lcode, 0, (size_t)m, st));
    JTB_OK(cudaMemsetAsync(p.srounds, 0, (size_t)S * 4, st));
    mono_scatter<<<grid((int64_t)m * 32, 256), 256, 0, st>>>(m, d.payload, poff, x.shard, x.inv, x.row, d.n_keys,
                                                             d.key_off, d.keys, V, key0, id0);
    size_t tb = tmp_bytes;
    JTB_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, key0, key1, id0, id1, m, MonoKeyDecomposer{}, st));
    if (nT > 0) {
        tl_tkeys<<<grid(nT, 256), 256, 0, st>>>(nT, d.t_shard, tid, tk0, tid0);
        tb = tmp_bytes;
        JTB_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, tk0, tk, tid0, tperm, nT, TlTKeyDecomposer{}, st));
    }
    if (nR > 0) {
        tl_records<<<grid(nR, 256), 256, 0, st>>>(d, rk0, rv0);
        tb = tmp_bytes;
        JTB_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, rk0, rk, rv0, rv, (int)nR, TlRKeyDecomposer{}, st));
    }
    if (nT > 0) {
        tl_mval<<<grid(nT, 256), 256, 0, st>>>(d, mk);
        rx_mark<<<grid(nT, 256), 256, 0, st>>>(d, tM, tA);
    }
    // the windows
    tp_pos<<<grid(m, 256), 256, 0, st>>>(m, id1, pos);
    tb = tmp_bytes;
    JTB_OK(cub::DeviceScan::InclusiveScan(tmp, tb, pos, cmax, MaxOp{}, m, st));
    tp_ivpos<<<grid(m, 256), 256, 0, st>>>(m, d_ivperm, pos, rev);
    tb = tmp_bytes;
    JTB_OK(cub::DeviceScan::InclusiveScan(tmp, tb, rev, srev, MinOp{}, m, st));
    if (nT > 0) tp_window<<<grid(nT, 256), 256, 0, st>>>(x, p, cmax, d_ivs, srev);
    // the rounds
    for (int32_t r = 0;; ++r) {
        if (r >= 2) {
            tb = tmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveSum(tmp, tb, p.dd, dirty, m + 1, st));
        }
        JTB_OK(cudaMemsetAsync(p.dd, 0, (size_t)(m + 1) * 4, st));
        JTB_OK(cudaMemsetAsync(x.f1, 0x7f, (size_t)nT * 4, st));
        JTB_OK(cudaMemsetAsync(x.f2, 0x7f, (size_t)nT * 4, st));
        JTB_OK(cudaMemsetAsync(p.pmin, 0x7f, (size_t)nT * 4, st));
        JTB_OK(cudaMemsetAsync(p.pmax, 0xff, (size_t)nT * 4, st));
        JTB_OK(cudaMemsetAsync(p.changed, 0, 4, st));
        p.round = r;
        tp_gaps<<<grid(m, RG_WARPS), RG_WARPS * 32, 0, st>>>(x, p);
        tp_possible<<<grid((int64_t)m * 32, 256), 256, 0, st>>>(m, p);
        tb = tmp_bytes;
        JTB_OK(cub::DeviceScan::InclusiveSum(tmp, tb, p.inc, incsum, m, st));
        if (nT > 0) tp_owner<<<grid(nT, 256), 256, 0, st>>>(x, p);
        JTB_OK(cudaGetLastError());
        unsigned int changed = 0;
        JTB_OK(cudaMemcpyAsync(&changed, p.changed, 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        if (r + 1 >= max_rounds || (r >= 1 && !changed)) break;
    }
    return 0;
}

// K12's finals over the stage's device state: the counts, the verdicts and the witnesses into shards[S] (filled with
// the verdicts of the shards the device does not run first); ev1 is recorded after the last kernel
inline int tp_finals(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, TpStage& g,
                     jtb_tp_shard* shards, float& ms, std::string& err) {
    const int32_t S = g.S;
    const MonoHost& H = g.H;
    const TlHost& T = g.T;
    for (int32_t s = 0; s < S; ++s) {
        jtb_tp_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_reads = H.n_reads[s];
        o.n_transfers = T.t_off[s + 1] - T.t_off[s];
        o.witness_index = o.lower_index = o.key = o.other_index = o.round = -1;
        if (H.n_reads[s] > 0 && !g.dev[s]) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_PARTIAL_READ;
        }
    }
    ms = 0;
    if (g.m == 0) return 0;
    const int32_t nT = g.nT;
    RgDev& x = g.x;
    TpDev& p = g.p;
    auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };
    tp_gap_final<<<grid(g.m, 256), 256, 0, st>>>(x, p);
    if (nT > 0) {
        tp_transfer_final<<<grid(nT, 256), 256, 0, st>>>(x, p);
        tp_witness_id<<<grid(nT, 256), 256, 0, st>>>(x, p);
    }
    JTB_OK(cudaGetLastError());
    JTB_OK(cudaEventRecord(ev1, st));
    std::vector<unsigned long long> cnt_h((size_t)S * TP_COUNTERS), wkey_h(S), wtid_h(S);
    std::vector<int32_t> sr_h(S);
    JTB_OK(cudaMemcpyAsync(cnt_h.data(), g.cnt, cnt_h.size() * 8, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaMemcpyAsync(wkey_h.data(), g.wkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaMemcpyAsync(wtid_h.data(), g.wtid, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaMemcpyAsync(sr_h.data(), p.srounds, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaStreamSynchronize(st));
    JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
    auto get = [&](auto* dst, const auto* src) {   // one scalar of a witness
        return cudaMemcpy(dst, src, sizeof *dst, cudaMemcpyDeviceToHost) == cudaSuccess;
    };
    auto index_at = [&](int32_t at) -> int32_t {   // completion :index of the read at a sorted position
        int32_t r;
        if (!get(&r, x.ord + at)) return INT_MIN;
        return h->index[H.r_ev[g.d_of[r]]];
    };
    for (int32_t s = 0; s < S; ++s) {
        jtb_tp_shard& o = shards[s];
        if (!g.dev[s]) continue;
        const unsigned long long* c = &cnt_h[(size_t)s * TP_COUNTERS];
        o.n_explained = (int64_t)c[0];
        o.n_undecided = (int64_t)c[1];
        for (int k = 0; k < 4; ++k) o.count_by_kind[k] = (int64_t)c[2 + k];
        o.n_placed = (int64_t)c[6];
        o.nodes = (int64_t)c[7];
        o.rounds = sr_h[s];
        if (wkey_h[s] != ~0ull) {
            const int32_t at = (int32_t)(wkey_h[s] >> 3);
            bool ok = true;
            o.kind = (int32_t)(wkey_h[s] & 7);
            o.witness_index = index_at(at);
            if (at > g.rs_off[s]) o.lower_index = index_at(at - 1);
            ok &= get(&o.n_eligible, x.gkept + at);
            if (o.kind == JTB_TP_DOUBLE || o.kind == JTB_TP_LOST) {
                o.transfer_id = (int64_t)(wtid_h[s] ^ 0x8000000000000000ull);
                int32_t t = T.t_off[s];
                while (T.t_id[t] != o.transfer_id) ++t;
                if (o.kind == JTB_TP_DOUBLE) {
                    int32_t first;
                    ok &= get(&o.round, p.dround + t) && get(&first, p.dg1 + t);
                    o.other_index = index_at(first);
                } else {
                    int32_t M;
                    ok &= get(&o.round, p.lround + t) && get(&M, g.tM + t);
                    o.other_index = h->index[h->shard_off[s] + M];
                }
            } else {
                ok &= get(&o.key, x.gkey + at) && get(&o.round, p.lround_g + at);
                if (o.kind == JTB_TP_KEY) ok &= get(&o.delta, x.gdelta + at);
            }
            if (!ok || o.witness_index == INT_MIN || o.lower_index == INT_MIN || o.other_index == INT_MIN) {
                err = "cudaMemcpy of a witness field failed";
                return -1;
            }
            o.valid = JTB_INVALID;
        } else if (o.n_undecided > 0) {
            o.valid = JTB_UNKNOWN;
        }
    }
    return 0;
}

inline int run_transfer_placement(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                                  int64_t max_nodes, int32_t max_rounds, int32_t flags, jtb_tp_shard* shards,
                                  jtb_tp_result* out, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    TpStage g;
    if (int rc = tp_stage(st, ev0, h, max_nodes, max_rounds, flags, g, err)) return rc;
    float ms = 0;
    if (int rc = tp_finals(st, ev0, ev1, h, g, shards, ms, err)) return rc;
    memset(out, 0, sizeof *out);
    for (int32_t s = 0; s < g.S; ++s) {
        const jtb_tp_shard& o = shards[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_explained += o.n_explained;
        out->n_unexplained += o.count_by_kind[0] + o.count_by_kind[1];
        out->n_double += o.count_by_kind[2];
        out->n_lost += o.count_by_kind[3];
        out->n_undecided += o.n_undecided;
        out->n_placed += o.n_placed;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
    }
    roll_up(out, shards, g.S, ms, t0);
    return 0;
}

}  // namespace jtb
