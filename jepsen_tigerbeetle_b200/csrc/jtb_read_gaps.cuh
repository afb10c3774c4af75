// jtb_read_gaps.cuh — K11: the read-gap check (do the transfers committed between two successive ledger reads explain
// what changed?) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K11 read-gap check").  The reads, the shards' key tables and the order of
// the reads are K7's: mono_host_pass, a dense row per read of a full-key shard (mono_scatter) and the stable radix
// sort by (shard, S as 128 bits, invocation).  The transfers, M(t) and A(t) are K9's and K10's, unchanged: the sort by
// (shard, id), tl_records, the sort of the records by (lookup, id), tl_mval and rx_mark.  Then:
//   - rg_gaps, a warp per sorted position i (the gap closed by the read there): Delta from two coalesced row reads
//     (the previous read of the shard in the order, or zero for gap 0); a negative component is KEY, Delta = 0 is
//     explained; otherwise the eligible transfers are gathered into shared memory with the amount filter applied
//     while gathering (the shard's :ok transfers in invocation order, back to the last one whose running max
//     completion precedes the lower read's invocation, and the crashed ones anchored at each key that grew, invoked
//     before the upper read completed), the transfers the root pruning forces in are recorded per transfer (the
//     smallest and the second smallest gap, by two atomicMin), and K10's rx_search decides the gap, key by key for
//     the kind of an unexplained one;
//   - rg_double and rg_double_witness, a thread per transfer: a transfer forced into two gaps is DOUBLE at the later
//     one; the shard's witness is the first violating gap with the smallest kind, a DOUBLE one the smallest id there.
// The decision, the caps and the node counts equal the RG_SEARCH CPU test oracle's, gap for gap.
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
#include "jtb_transfer_lookups.cuh"

namespace jtb {

static_assert(JTB_RG_MAX_KEYS == JTB_RX_MAX_KEYS && JTB_RG_MAX_GATHER == JTB_RX_MAX_GATHER &&
                  JTB_RG_MAX_FREE == JTB_RX_MAX_FREE, "K11 runs K10's search on K10's shared-memory layout");

constexpr int RG_WARPS = 4;   // warps per block of rg_gaps
constexpr int RG_COUNTERS = 6;   // per shard: explained, undecided, KEY, JOINT, DOUBLE, nodes
constexpr int32_t RG_NONE = 0x7f7f7f7f;   // no gap (the memset byte 0x7f; more gaps than that do not fit a device)

struct RgDev {
    // reads of the full-key shards (device ids in completion order) and their order
    int32_t m = 0;
    const int32_t* ord = nullptr;         // [m] device read ids in gap order
    const int32_t* shard = nullptr;
    const int32_t* inv = nullptr;         // -1 = none
    const int32_t* comp = nullptr;
    const int64_t* row = nullptr;         // offset of the read's row in V
    const int64_t* V = nullptr;
    const int32_t* n_keys = nullptr;
    const int64_t* key_off = nullptr;
    const int32_t* keys = nullptr;
    // transfers, in K9's order (shard-major, invocation order)
    const int32_t* t_rec = nullptr;       // (debit, credit, amount) x n_t
    const int64_t* t_id = nullptr;
    const int32_t* t_M = nullptr;
    const int32_t* t_A = nullptr;
    // the shard's :ok transfers by invocation with the running max of their completions; the crashed ones by
    // invocation, grouped by anchor slot (key_off[s] + the column of the debit key, or of the credit key when no read
    // observes the debit key)
    const int32_t* ok_t = nullptr;
    const int32_t* ok_inv = nullptr;
    const int32_t* ok_pmax = nullptr;
    const int32_t* ok_off = nullptr;      // [n_shards + 1]
    const int32_t* cr_t = nullptr;
    const int32_t* cr_inv = nullptr;
    const int32_t* cr_off = nullptr;      // [slots + 1]
    int64_t max_nodes = 0;
    // per transfer: the smallest and the second smallest gap that forces it in, RG_NONE none
    int32_t* f1 = nullptr;
    int32_t* f2 = nullptr;
    // per gap (sorted position)
    int8_t* code = nullptr;
    int32_t* gkey = nullptr;
    int32_t* gkept = nullptr;
    int64_t* gdelta = nullptr;
    // per shard
    unsigned long long* cnt = nullptr;    // [n_shards * RG_COUNTERS]
    unsigned long long* wkey = nullptr;   // [n_shards] min of gap << 2 | kind
    unsigned long long* wtid = nullptr;   // [n_shards] min of id ^ 2^63 of the DOUBLE transfers at the witness gap
};

// one warp's shared state: K10's, plus the transfer of each gathered candidate
struct RgWarp {
    RxWarp x;
    int32_t ct[JTB_RG_MAX_GATHER];
};

// The gather of the gap closed by a read completed at cp over the previous read invoked at ivl (-1 for gap 0), Delta
// and the keys in W: the shard's eligible transfers that fit under Delta and pass extra(t), into the candidate arrays
// of W and G.ct.  Returns how many there are; more than JTB_RG_MAX_GATHER means the gap has too many (the arrays hold
// the first ones).  cap(valid, t, amount, jd, jc, n), called by the whole warp on every batch of crashed transfers,
// may drop more of them (the class witness's per-class cap); the default keeps them.
struct RgNoCap {
    __device__ __forceinline__ bool operator()(bool valid, int32_t, int32_t, int16_t, int16_t, int32_t) const {
        return valid;
    }
};

template <class Extra, class Cap = RgNoCap>
__device__ __forceinline__ int32_t rg_gather(const RgDev& d, RgWarp& G, int32_t s, int32_t K, int32_t cp, int32_t ivl,
                                             int lane, Extra extra, Cap cap = {}) {
    RxWarp& W = G.x;
    int32_t n = 0;
    auto find = [&](int64_t k) {
        int32_t a = 0, b = K;
        while (a < b) {
            const int32_t c = (a + b) >> 1;
            if (W.key[c] < k) a = c + 1; else b = c;
        }
        return (int16_t)(a < K && W.key[a] == k ? a : -1);
    };
    auto take = [&](bool valid, int32_t t, auto capped) {
        int16_t jd = -1, jc = -1;
        int32_t a = 0;
        if (valid) {
            const int32_t* q = d.t_rec + 3 * (int64_t)t;
            a = q[2];
            valid = !(d.t_M[t] < ivl) && d.t_A[t] < cp && a > 0 && extra(t);
            if (valid) {
                jd = find(2 * (int64_t)q[0]);
                jc = find(2 * (int64_t)q[1] + 1);
                valid = (jd >= 0 || jc >= 0) && (jd < 0 || a <= W.d[jd]) && (jc < 0 || a <= W.d[jc]);
            }
        }
        valid = capped(valid, t, a, jd, jc, n);
        const unsigned bal = __ballot_sync(0xffffffffu, valid);
        const int32_t at = n + __popc(bal & ((1u << lane) - 1));
        if (valid && at < JTB_RG_MAX_GATHER) {
            W.cid[at] = d.t_id[t];
            W.ca[at] = a;
            W.cjd[at] = jd;
            W.cjc[at] = jc;
            G.ct[at] = t;
        }
        n += __popc(bal);
    };
    const int32_t olo = d.ok_off[s], b = rx_lower(d.ok_inv, olo, d.ok_off[s + 1], cp);
    for (int32_t base = b - 1; base >= olo && n <= JTB_RG_MAX_GATHER; base -= 32) {
        const int32_t j = base - lane;
        const bool valid = j >= olo && d.ok_pmax[j] >= ivl;
        if (!__any_sync(0xffffffffu, valid)) break;
        take(valid, valid ? d.ok_t[j] : 0, RgNoCap{});
    }
    for (int32_t c = 0; c < K && n <= JTB_RG_MAX_GATHER; ++c) {
        if (W.d[c] <= 0) continue;   // a crashed transfer anchored at c needs its amount <= Delta_c
        const int64_t slot = d.key_off[s] + c;
        const int32_t clo = d.cr_off[slot], bc = rx_lower(d.cr_inv, clo, d.cr_off[slot + 1], cp);
        for (int32_t base = clo; base < bc && n <= JTB_RG_MAX_GATHER; base += 32) {
            const int32_t j = base + lane;
            take(j < bc, j < bc ? d.cr_t[j] : 0, cap);
        }
    }
    return n;
}

// warp per gap
__global__ void __launch_bounds__(RG_WARPS * 32) rg_gaps(RgDev d) {
    __shared__ RgWarp smem[RG_WARPS];
    const int lane = threadIdx.x & 31;
    RgWarp& G = smem[threadIdx.x >> 5];
    RxWarp& W = G.x;
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (w >= d.m) return;
    const int32_t i = (int32_t)w, u = d.ord[i], s = d.shard[u], K = d.n_keys[s], cp = d.comp[u];
    const int32_t lower = i > 0 && d.shard[d.ord[i - 1]] == s ? d.ord[i - 1] : -1;
    const int32_t ivl = lower >= 0 ? d.inv[lower] : -1;   // M(t) >= 0 > -1: gap 0 drops nothing by M
    int8_t code = RX_UNDECIDED;
    int64_t nodes = 0, delta = 0;
    int32_t gkey = -1, kept = 0;
    if (K <= JTB_RG_MAX_KEYS) {
        const int64_t* vu = d.V + d.row[u];
        const int64_t* vl = lower >= 0 ? d.V + d.row[lower] : nullptr;
        const int32_t* kt = d.keys + d.key_off[s];
        int32_t neg = INT_MAX;
        bool nz = false;
        for (int32_t j = lane; j < K; j += 32) {
            const int64_t x = vu[j] - (vl ? vl[j] : 0);
            W.key[j] = kt[j];
            W.d[j] = x;
            if (x < 0) neg = min(neg, j);
            nz |= x != 0;
        }
        neg = rx_warp_min(neg);
        nz = __any_sync(0xffffffffu, nz);
        __syncwarp();
        if (neg != INT_MAX) {
            code = JTB_RG_KEY;
            gkey = W.key[neg];
            delta = W.d[neg];
        } else if (!nz) {
            code = RX_EXPLAINED;
        } else {
            // gather the eligible transfers that fit under Delta; n > cap = too many
            const int32_t n = rg_gather(d, G, s, K, cp, ivl, lane, [](int32_t) { return true; });
            __syncwarp();
            if (n <= JTB_RG_MAX_GATHER) {
                // the root pruning once more, as rx_search starts, to record the transfers it forces in
                for (int32_t c = lane; c < n; c += 32) {
                    W.idx[c] = (uint8_t)c;
                    W.st[c] = RX_UND;
                }
                __syncwarp();
                int32_t bad;
                if (rx_prune(W, K, n, -1, lane, bad))
                    for (int32_t c = lane; c < n; c += 32) {
                        if (W.st[c] != RX_IN) continue;
                        const int32_t t = G.ct[c], old = atomicMin(&d.f1[t], i);
                        if (old != RG_NONE) atomicMin(&d.f2[t], max(old, i));
                    }
                __syncwarp();
                int32_t root_key;
                code = (int8_t)rx_search(W, K, n, -1, d.max_nodes, lane, nodes, root_key, kept);
                if (code == JTB_RG_JOINT) {
                    gkey = root_key;
                    for (int32_t k = 0; k < K; ++k) {
                        int32_t rk, kp;
                        if (rx_search(W, K, n, k, d.max_nodes, lane, nodes, rk, kp) == JTB_RG_JOINT) {
                            code = JTB_RG_KEY;
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
    unsigned long long* c = d.cnt + (int64_t)s * RG_COUNTERS;
    atomicAdd(&c[5], (unsigned long long)nodes);
    d.gkept[i] = kept;
    if (code == RX_EXPLAINED) { atomicAdd(&c[0], 1ull); return; }
    if (code == RX_UNDECIDED) { atomicAdd(&c[1], 1ull); return; }
    atomicAdd(&c[1 + code], 1ull);
    atomicMin(&d.wkey[s], (unsigned long long)i << 2 | (unsigned)code);
    d.code[i] = code;
    d.gkey[i] = gkey;
    d.gdelta[i] = delta;
}

// thread per transfer: one forced into two gaps is DOUBLE at the later of the two smallest
__global__ void rg_double(int32_t n_t, const int32_t* __restrict__ t_shard, const int32_t* __restrict__ f2,
                          unsigned long long* __restrict__ cnt, unsigned long long* __restrict__ wkey) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_t || f2[t] == RG_NONE) return;
    const int32_t s = t_shard[t];
    atomicAdd(&cnt[(int64_t)s * RG_COUNTERS + 4], 1ull);
    atomicMin(&wkey[s], (unsigned long long)f2[t] << 2 | JTB_RG_DOUBLE);
}

// thread per transfer: the smallest id among the DOUBLE transfers at their shard's witness gap
__global__ void rg_double_witness(int32_t n_t, const int32_t* __restrict__ t_shard, const int64_t* __restrict__ t_id,
                                  const int32_t* __restrict__ f2, const unsigned long long* __restrict__ wkey,
                                  unsigned long long* __restrict__ wtid) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_t || f2[t] == RG_NONE) return;
    const int32_t s = t_shard[t];
    if (wkey[s] == ((unsigned long long)f2[t] << 2 | JTB_RG_DOUBLE))
        atomicMin(&wtid[s], (unsigned long long)t_id[t] ^ 0x8000000000000000ull);
}

// ---- host ---------------------------------------------------------------------------------------------------------

inline int run_read_gaps(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, int64_t max_nodes,
                         int32_t flags, jtb_rg_shard* shards, jtb_rg_result* out, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    if (flags != 0) { err = "flags must be 0 (reserved)"; return -2; }
    if (int rc = check_history(h, false, err)) return rc;
    if (max_nodes <= 0) max_nodes = JTB_RG_DEFAULT_MAX_NODES;
    const int32_t S = h->n_shards;
    MonoHost H;
    if (int rc = mono_host_pass(h, H, err)) return rc;
    TlHost T;
    if (int rc = tl_host_pass(h, T, err)) return rc;
    if (T.t_id.size() > (size_t)1 << 30) { err = "more than 2^30 transfers"; return -2; }
    const int32_t nT = (int32_t)T.t_id.size(), nL = (int32_t)T.l_shard.size();
    const int64_t nR = T.rec_base.back(), slots = (int64_t)H.keys.size();
    memset(out, 0, sizeof *out);
    std::vector<char> dev(S, 0);
    for (int32_t s = 0; s < S; ++s) {
        jtb_rg_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_reads = H.n_reads[s];
        o.n_transfers = T.t_off[s + 1] - T.t_off[s];
        o.witness_index = o.lower_index = o.key = o.other_index = -1;
        if (H.n_reads[s] > 0 && H.min_trip[s] < H.n_keys[s]) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_PARTIAL_READ;
        } else if (H.n_reads[s] > 0) dev[s] = 1;
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
    }
    // the device's reads (ids compacted over the full-key shards, as K7 does) and their rows
    std::vector<int32_t> d_of, shard_v, inv_v, comp_v;
    std::vector<int64_t> poff_v, row_v;
    int64_t cells = 0;
    for (int32_t r = 0; r < (int32_t)H.r_shard.size(); ++r) {
        const int32_t s = H.r_shard[r];
        if (!dev[s]) continue;
        d_of.push_back(r);
        shard_v.push_back(s);
        inv_v.push_back(H.r_inv[r]);
        comp_v.push_back(H.r_comp[r]);
        poff_v.push_back(H.r_poff[r]);
        row_v.push_back(cells);
        cells += H.n_keys[s];
    }
    const int32_t m = (int32_t)d_of.size();
    // the :ok transfers of every shard by invocation (the order of T), and the crashed ones by anchor slot
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
    for (int32_t t = 0; t < nT; ++t)   // T's order: invocation order inside every slot
        if (cr_anchor[t] >= 0) {
            const int32_t j = fill[cr_anchor[t]]++;
            cr_t[j] = t;
            cr_inv[j] = T.t_inv[t];
        }
    float ms = 0;
    if (m > 0) {
        CallAllocs A;
        int64_t* V;
        if (A.alloc(&V, (size_t)cells) != cudaSuccess) {
            err = "cannot allocate the dense value matrix (" + std::to_string((size_t)cells * sizeof(int64_t)) +
                  " bytes on the device)";
            return -3;
        }
        TlDev d;
        RgDev x;
        d.n_t = nT;
        d.n_l = nL;
        d.n_rec = nR;
        x.m = m;
        x.V = V;
        x.max_nodes = max_nodes;
        const int64_t* tid;
        const int64_t* poff;
        TlTKey *tk0, *tk;
        TlRKey *rk0, *rk;
        MonoKey *key0, *key1;
        int32_t *tid0, *tperm, *rv0, *rv, *tM, *tA, *id0, *id1;
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
        JTB_OK(A.alloc(&key0, m)); JTB_OK(A.alloc(&key1, m)); JTB_OK(A.alloc(&id0, m)); JTB_OK(A.alloc(&id1, m));
        JTB_OK(A.alloc(&tk0, nT)); JTB_OK(A.alloc(&tk, nT)); JTB_OK(A.alloc(&tid0, nT)); JTB_OK(A.alloc(&tperm, nT));
        JTB_OK(A.alloc(&d.rec_slot, nR)); JTB_OK(A.alloc(&rk0, nR)); JTB_OK(A.alloc(&rk, nR));
        JTB_OK(A.alloc(&rv0, nR)); JTB_OK(A.alloc(&rv, nR));
        JTB_OK(A.alloc(&d.mlk, nT)); JTB_OK(A.alloc(&d.mv, nT)); JTB_OK(A.alloc(&d.mfrom, nT)); JTB_OK(A.alloc(&mk, nT));
        JTB_OK(A.alloc(&d.wid, (size_t)nL * 5)); JTB_OK(A.alloc(&d.count, (size_t)S * JTB_TL_KINDS));
        JTB_OK(A.alloc(&tM, nT)); JTB_OK(A.alloc(&tA, nT)); JTB_OK(A.alloc(&x.f1, nT)); JTB_OK(A.alloc(&x.f2, nT));
        JTB_OK(A.alloc(&x.code, m)); JTB_OK(A.alloc(&x.gkey, m)); JTB_OK(A.alloc(&x.gkept, m));
        JTB_OK(A.alloc(&x.gdelta, m));
        JTB_OK(A.alloc(&cnt, (size_t)S * RG_COUNTERS)); JTB_OK(A.alloc(&wkey, S)); JTB_OK(A.alloc(&wtid, S));
        d.tkey = tk; d.tperm = tperm; d.rkey = rk; d.rval = rv;
        x.ord = id1; x.t_M = tM; x.t_A = tA; x.cnt = cnt; x.wkey = wkey; x.wtid = wtid;
        size_t tmp_m = 0, tmp_t = 0, tmp_r = 0;
        JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_m, key0, key1, id0, id1, m, MonoKeyDecomposer{}, st));
        if (nT > 0)
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_t, tk0, tk, tid0, tperm, nT, TlTKeyDecomposer{}, st));
        if (nR > 0)
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_r, rk0, rk, rv0, rv, (int)nR, TlRKeyDecomposer{}, st));
        const size_t tmp_bytes = std::max({tmp_m, tmp_t, tmp_r});
        JTB_OK(A.alloc(&tmp, tmp_bytes));
        auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };

        JTB_OK(cudaEventRecord(ev0, st));
        JTB_OK(cudaMemsetAsync(d.mlk, 0x7f, (size_t)nT * 4, st));   // 0x7f7f7f7f > any lookup id: "none"
        JTB_OK(cudaMemsetAsync(d.wid, 0xff, (size_t)nL * 40, st));
        JTB_OK(cudaMemsetAsync(d.count, 0, (size_t)S * JTB_TL_KINDS * 8, st));
        JTB_OK(cudaMemsetAsync(x.f1, 0x7f, (size_t)nT * 4, st));   // RG_NONE
        JTB_OK(cudaMemsetAsync(x.f2, 0x7f, (size_t)nT * 4, st));
        JTB_OK(cudaMemsetAsync(cnt, 0, (size_t)S * RG_COUNTERS * 8, st));
        JTB_OK(cudaMemsetAsync(wkey, 0xff, (size_t)S * 8, st));
        JTB_OK(cudaMemsetAsync(wtid, 0xff, (size_t)S * 8, st));
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
        rg_gaps<<<grid(m, RG_WARPS), RG_WARPS * 32, 0, st>>>(x);
        if (nT > 0) {
            rg_double<<<grid(nT, 256), 256, 0, st>>>(nT, d.t_shard, x.f2, cnt, wkey);
            rg_double_witness<<<grid(nT, 256), 256, 0, st>>>(nT, d.t_shard, tid, x.f2, wkey, wtid);
        }
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<unsigned long long> cnt_h((size_t)S * RG_COUNTERS), wkey_h(S), wtid_h(S);
        JTB_OK(cudaMemcpyAsync(cnt_h.data(), cnt, cnt_h.size() * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(wkey_h.data(), wkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(wtid_h.data(), wtid, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        auto index_at = [&](int32_t pos) -> int32_t {   // completion :index of the read at a sorted position
            int32_t r;
            if (cudaMemcpy(&r, id1 + pos, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return INT_MIN;
            return h->index[H.r_ev[d_of[r]]];
        };
        for (int32_t s = 0; s < S; ++s) {
            jtb_rg_shard& o = shards[s];
            if (!dev[s]) continue;
            const unsigned long long* c = &cnt_h[(size_t)s * RG_COUNTERS];
            o.n_explained = (int64_t)c[0];
            o.n_undecided = (int64_t)c[1];
            for (int k = 0; k < 3; ++k) o.count_by_kind[k] = (int64_t)c[2 + k];
            o.nodes = (int64_t)c[5];
            if (wkey_h[s] != ~0ull) {   // the witness gap's fields: a few scalars per INVALID shard
                const int32_t pos = (int32_t)(wkey_h[s] >> 2);
                o.kind = (int32_t)(wkey_h[s] & 3);
                o.witness_index = index_at(pos);
                int32_t prev = -1;
                if (pos > 0) JTB_OK(cudaMemcpy(&prev, id1 + pos - 1, 4, cudaMemcpyDeviceToHost));
                if (pos > 0 && shard_v[prev] == s) o.lower_index = index_at(pos - 1);
                JTB_OK(cudaMemcpy(&o.n_eligible, x.gkept + pos, 4, cudaMemcpyDeviceToHost));
                if (o.kind == JTB_RG_DOUBLE) {
                    o.transfer_id = (int64_t)(wtid_h[s] ^ 0x8000000000000000ull);
                    int32_t t = T.t_off[s];
                    while (T.t_id[t] != o.transfer_id) ++t;
                    int32_t first;
                    JTB_OK(cudaMemcpy(&first, x.f1 + t, 4, cudaMemcpyDeviceToHost));
                    o.other_index = index_at(first);
                } else {
                    JTB_OK(cudaMemcpy(&o.key, x.gkey + pos, 4, cudaMemcpyDeviceToHost));
                    if (o.kind == JTB_RG_KEY) JTB_OK(cudaMemcpy(&o.delta, x.gdelta + pos, 8, cudaMemcpyDeviceToHost));
                }
                if (o.witness_index == INT_MIN || o.lower_index == INT_MIN || o.other_index == INT_MIN) {
                    err = "cudaMemcpy of a witness read failed";
                    return -1;
                }
                o.valid = JTB_INVALID;
            } else if (o.n_undecided > 0) {
                o.valid = JTB_UNKNOWN;
            }
        }
    }
    for (int32_t s = 0; s < S; ++s) {
        const jtb_rg_shard& o = shards[s];
        out->n_explained += o.n_explained;
        out->n_unexplained += o.count_by_kind[0] + o.count_by_kind[1];
        out->n_double += o.count_by_kind[2];
        out->n_undecided += o.n_undecided;
        out->nodes += o.nodes;
    }
    roll_up(out, shards, S, ms, t0);
    return 0;
}

}  // namespace jtb
