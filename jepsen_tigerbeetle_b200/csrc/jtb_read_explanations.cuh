// jtb_read_explanations.cuh — K10: the read-explanation check (does one set of transfers explain every counter an :ok
// ledger read shows?) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K10 read-explanation check").  The reads and the shards' key tables are
// K7's host pass (mono_host_pass), the transfers and lookups K9's (tl_host_pass), and K9's first kernels give every
// transfer M(t): the sort by (shard, id), tl_records, the sort of the records by (lookup, id) and tl_mval.  Then:
//   - rx_mark, a thread per transfer: M and A(t), the latest invocation of an :ok lookup lacking t (a binary search per
//     lookup, latest invocation first, in the records sorted by (lookup, id));
//   - rx_contrib and a radix sort of (slot << 32 | M) with the amounts, then an inclusive sum by slot: the must sum of
//     a (read, key) is one prefix of its slot, found by binary search (K8's layout with M in place of the completion);
//   - rx_reads, a warp per read: the read's keys sorted into shared memory with d_k = v_k - must_k, the "may"
//     transfers gathered into shared memory (the shard's :ok transfers in invocation order, back to the last one whose
//     running max completion precedes the read's invocation, and its crashed transfers invoked before the read
//     completed), the root pruning fixpoint in Jacobi rounds with per-key sums by shared atomics, then the canonical
//     depth-first search over at most 64 free candidates as two 64-bit masks, re-pruning at every node; an unexplained
//     read is searched again key by key for its kind;
//   - rx_must_count, a thread per transfer: |must| of each shard's witness read; the host copies back the few scalars
//     rx_reads left for that read.
// The decision, the caps and the node counts equal the RX_SEARCH CPU test oracle's, read for read.
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
#include "jtb_counter_bounds.cuh"
#include "jtb_monotonic.cuh"
#include "jtb_transfer_lookups.cuh"

namespace jtb {

constexpr int RX_WARPS = 4;   // warps per block of rx_reads
constexpr uint8_t RX_UND = 0, RX_IN = 1, RX_OUT = 2;
constexpr int8_t RX_EXPLAINED = 0, RX_UNDECIDED = 3;   // per-read codes; 1 / 2 are JTB_RX_KEY / JTB_RX_JOINT

struct RxDev {
    const int32_t* payload = nullptr;
    // reads (K7's)
    int32_t m = 0;
    const int64_t* poff = nullptr;
    const int32_t* ntrip = nullptr;
    const int32_t* r_shard = nullptr;
    const int32_t* r_inv = nullptr;
    const int32_t* r_comp = nullptr;
    const int32_t* n_keys = nullptr;
    const int64_t* key_off = nullptr;
    const int32_t* keys = nullptr;
    // transfers, in K9's order (shard-major, invocation order)
    int32_t n_t = 0;
    const int32_t* t_shard = nullptr;
    const int32_t* t_rec = nullptr;       // (debit, credit, amount) x n_t
    const int64_t* t_id = nullptr;
    const int32_t* t_M = nullptr;
    const int32_t* t_A = nullptr;
    // the shard's :ok transfers (with the running max of their completions) and crashed ones, by invocation
    const int32_t* ok_t = nullptr;
    const int32_t* ok_inv = nullptr;
    const int32_t* ok_pmax = nullptr;
    const int32_t* ok_off = nullptr;      // [n_shards + 1]
    const int32_t* cr_t = nullptr;
    const int32_t* cr_inv = nullptr;
    const int32_t* cr_off = nullptr;      // [n_shards + 1]
    // must sums: (slot << 32 | M) sorted, inclusive sums of the amounts by slot
    int32_t n_c = 0;
    const uint64_t* ckey = nullptr;
    const int64_t* csum = nullptr;
    int64_t max_nodes = 0;
    // per read
    int8_t* code = nullptr;
    int32_t* rkey = nullptr;
    int32_t* rmay = nullptr;
    int64_t* rvalue = nullptr;
    int64_t* rmust = nullptr;
    // per shard
    unsigned long long* cnt = nullptr;    // [n_shards * 5]: explained, undecided, KEY, JOINT, nodes
    unsigned long long* wread = nullptr;  // [n_shards] the smallest unexplained read id
    int32_t* nmust = nullptr;             // [n_shards]
};

// thread per transfer slot: M and A(t) by original transfer
__global__ void rx_mark(TlDev d, int32_t* __restrict__ tM, int32_t* __restrict__ tA) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.n_t) return;
    const int32_t t = d.tperm[i], s = d.t_shard[t];
    const uint64_t idu = d.tkey[i].idu;
    int32_t A = -1;
    for (int32_t j = d.ib_off[s + 1] - 1; j >= d.ib_off[s] && A < 0; --j) {
        const int32_t l = d.ib[j];
        int64_t a = d.rec_base[l], b = d.rec_base[l + 1];
        while (a < b) {
            const int64_t c = (a + b) >> 1;
            if (d.rkey[c].idu < idu) a = c + 1; else b = c;
        }
        if (!(a < d.rec_base[l + 1] && d.rkey[a].idu == idu)) A = d.ib_inv[j];
    }
    tM[t] = d.mv[i];
    tA[t] = A;
}

// thread per transfer: its two contributions (slot << 32 | M, amount); slot n_slots when no read observes the key
__global__ void rx_contrib(TlDev d, int32_t n_slots, const int32_t* __restrict__ tM, uint64_t* __restrict__ key,
                           int64_t* __restrict__ amt) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= d.n_t) return;
    const int32_t s = d.t_shard[t];
    const int32_t* q = d.t_rec + 3 * t;
    for (int side = 0; side < 2; ++side) {
        const int32_t col = tl_col(d, s, 2 * (int64_t)q[side] + side);
        const uint32_t slot = col >= 0 ? (uint32_t)(d.key_off[s] + col) : (uint32_t)n_slots;
        key[2 * t + side] = (uint64_t)slot << 32 | (uint32_t)tM[t];
        amt[2 * t + side] = q[2];
    }
}

// the must sum of slot for a read invoked at iv: the contributions with M < iv
__device__ __forceinline__ int64_t rx_must(const RxDev& d, int32_t slot, int32_t iv) {
    if (iv < 0) return 0;
    const uint64_t base = (uint64_t)(uint32_t)slot << 32;
    const int32_t lo = tl_lower(d.ckey, 0, d.n_c, base), hi = tl_lower(d.ckey, lo, d.n_c, base | (uint32_t)iv);
    return hi > lo ? d.csum[hi - 1] : 0;
}

// first j in [a, b) with v[j] >= x
__device__ __forceinline__ int32_t rx_lower(const int32_t* v, int32_t a, int32_t b, int32_t x) {
    while (a < b) {
        const int32_t c = (int32_t)(((int64_t)a + b) >> 1);
        if (v[c] < x) a = c + 1; else b = c;
    }
    return a;
}

// one warp's shared state
struct RxWarp {
    int64_t d[JTB_RX_MAX_KEYS];       // d_k by sorted key
    int64_t ins[JTB_RX_MAX_KEYS];     // per round: the sums of the IN / undecided candidates
    int64_t av[JTB_RX_MAX_KEYS];
    int64_t cid[JTB_RX_MAX_GATHER];
    uint64_t stk_in[JTB_RX_MAX_FREE], stk_out[JTB_RX_MAX_FREE];
    int32_t key[JTB_RX_MAX_KEYS];
    int32_t ca[JTB_RX_MAX_GATHER];
    int16_t cjd[JTB_RX_MAX_GATHER], cjc[JTB_RX_MAX_GATHER];
    uint8_t st[JTB_RX_MAX_GATHER];    // status by position of the list being pruned
    uint8_t idx[JTB_RX_MAX_GATHER];   // the list: candidate of each position
};

__device__ __forceinline__ int32_t rx_warp_min(int32_t x) {
    for (int o = 16; o; o >>= 1) x = min(x, __shfl_xor_sync(0xffffffffu, x, o));
    return x;
}
__device__ __forceinline__ int32_t rx_warp_sum(int32_t x) {
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// key index j relevant to a search over key `only` (-1: every key)
__device__ __forceinline__ int32_t rx_rel(int32_t j, int32_t only) { return only < 0 || j == only ? j : -1; }

// The pruning fixpoint in Jacobi rounds over list positions [0, cnt) (candidate W.idx[i], status W.st[i]).  false:
// infeasible, bad = the smallest infeasible key index of that round.
__device__ bool rx_prune(RxWarp& W, int32_t nt, int32_t cnt, int32_t only, int lane, int32_t& bad) {
    for (;;) {
        for (int32_t j = lane; j < nt; j += 32)
            if (rx_rel(j, only) >= 0) { W.ins[j] = 0; W.av[j] = 0; }
        __syncwarp();
        for (int32_t i = lane; i < cnt; i += 32) {
            const uint8_t s = W.st[i];
            if (s == RX_OUT) continue;
            const int32_t c = W.idx[i], kd = rx_rel(W.cjd[c], only), kc = rx_rel(W.cjc[c], only);
            int64_t* v = s == RX_IN ? W.ins : W.av;
            if (kd >= 0) atomicAdd((unsigned long long*)&v[kd], (unsigned long long)W.ca[c]);
            if (kc >= 0) atomicAdd((unsigned long long*)&v[kc], (unsigned long long)W.ca[c]);
        }
        __syncwarp();
        int32_t b = INT_MAX;
        for (int32_t j = lane; j < nt; j += 32) {
            if (rx_rel(j, only) < 0) continue;
            const int64_t need = W.d[j] - W.ins[j];
            if (need < 0 || need > W.av[j]) b = min(b, j);
        }
        b = rx_warp_min(b);
        if (b != INT_MAX) { bad = b; return false; }
        bool changed = false;
        for (int32_t i = lane; i < cnt; i += 32) {
            if (W.st[i] != RX_UND) continue;
            const int32_t c = W.idx[i];
            const int32_t ks[2] = {rx_rel(W.cjd[c], only), rx_rel(W.cjc[c], only)};
            const int64_t a = W.ca[c];
            bool drop = false, force = false;
            for (int32_t k : ks)
                if (k >= 0 && a > W.d[k] - W.ins[k]) drop = true;
            for (int32_t k : ks)
                if (!drop && k >= 0 && W.av[k] - a < W.d[k] - W.ins[k]) force = true;
            if (drop || force) { W.st[i] = drop ? RX_OUT : RX_IN; changed = true; }
        }
        changed = __any_sync(0xffffffffu, changed);
        __syncwarp();
        if (!changed) return true;
    }
}

// One search over the n gathered candidates (only >= 0: key `only` alone).  Returns RX_EXPLAINED, JTB_RX_JOINT
// (unexplained) or RX_UNDECIDED; adds its nodes; root_key / kept as in RX_SEARCH.
__device__ int rx_search(RxWarp& W, int32_t nt, int32_t n, int32_t only, int64_t max_nodes, int lane, int64_t& nodes,
                         int32_t& root_key, int32_t& kept) {
    for (int32_t c = lane; c < n; c += 32) {
        W.idx[c] = (uint8_t)c;
        W.st[c] = rx_rel(W.cjd[c], only) < 0 && rx_rel(W.cjc[c], only) < 0 ? RX_OUT : RX_UND;
    }
    __syncwarp();
    nodes += 1;   // the root; max_nodes counts down what is left
    --max_nodes;
    root_key = -1;
    int32_t bad;
    const bool ok = rx_prune(W, nt, n, only, lane, bad);
    int32_t nk = 0, nf = 0;
    for (int32_t c = lane; c < n; c += 32) { nk += W.st[c] != RX_OUT; nf += W.st[c] == RX_UND; }
    kept = rx_warp_sum(nk);
    nf = rx_warp_sum(nf);
    if (!ok) { root_key = W.key[bad]; return JTB_RX_JOINT; }
    if (nf == 0) return RX_EXPLAINED;
    if (nf > JTB_RX_MAX_FREE) return RX_UNDECIDED;
    // the list: the free candidates in the canonical order (amount descending, then id) at [0, nf), the forced ones
    // after them, IN for good
    uint8_t pos[JTB_RX_MAX_GATHER / 32];
    for (int32_t c = lane, q = 0; c < n; c += 32, ++q) {
        pos[q] = 0xff;
        if (W.st[c] == RX_OUT) continue;
        int32_t r = 0;
        if (W.st[c] == RX_UND) {
            for (int32_t o = 0; o < n; ++o)
                r += W.st[o] == RX_UND && (W.ca[o] > W.ca[c] || (W.ca[o] == W.ca[c] && W.cid[o] < W.cid[c]));
        } else {
            r = nf;
            for (int32_t o = 0; o < c; ++o) r += W.st[o] == RX_IN;
        }
        pos[q] = (uint8_t)r;
    }
    __syncwarp();
    for (int32_t c = lane, q = 0; c < n; c += 32, ++q)
        if (pos[q] != 0xff) W.idx[pos[q]] = (uint8_t)c;
    __syncwarp();
    const uint64_t full = nf == 64 ? ~0ull : (1ull << nf) - 1;
    uint64_t in = 0, out = 0;
    int32_t top = 0;
    for (;;) {
        const int32_t b = __ffsll((long long)(full & ~(in | out))) - 1;   // the state is pruned, feasible, not closed
        if (lane == 0) { W.stk_in[top] = in; W.stk_out[top] = out | 1ull << b; }
        ++top;
        in |= 1ull << b;
        for (;;) {
            if (++nodes, --max_nodes < 0) return RX_UNDECIDED;
            for (int32_t i = lane; i < kept; i += 32)
                W.st[i] = i >= nf ? RX_IN : (in >> i & 1) ? RX_IN : (out >> i & 1) ? RX_OUT : RX_UND;
            __syncwarp();
            if (rx_prune(W, nt, kept, only, lane, bad)) {
                const bool a = lane < nf && W.st[lane] == RX_IN, b2 = lane + 32 < nf && W.st[lane + 32] == RX_IN;
                const bool c = lane < nf && W.st[lane] == RX_OUT, d2 = lane + 32 < nf && W.st[lane + 32] == RX_OUT;
                in = (uint64_t)__ballot_sync(0xffffffffu, a) | (uint64_t)__ballot_sync(0xffffffffu, b2) << 32;
                out = (uint64_t)__ballot_sync(0xffffffffu, c) | (uint64_t)__ballot_sync(0xffffffffu, d2) << 32;
                if ((full & ~(in | out)) == 0) return RX_EXPLAINED;
                break;
            }
            if (top == 0) return JTB_RX_JOINT;
            --top;
            in = W.stk_in[top];
            out = W.stk_out[top];
            __syncwarp();
        }
    }
}

// warp per read
__global__ void __launch_bounds__(RX_WARPS * 32) rx_reads(RxDev d) {
    __shared__ RxWarp smem[RX_WARPS];
    const int lane = threadIdx.x & 31;
    RxWarp& W = smem[threadIdx.x >> 5];
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (w >= d.m) return;
    const int32_t r = (int32_t)w, s = d.r_shard[r], nt = d.ntrip[r], iv = d.r_inv[r], cp = d.r_comp[r];
    int8_t code = RX_UNDECIDED;
    int64_t nodes = 0;
    int32_t rkey = -1, kept = 0, n = 0;
    if (nt <= JTB_RX_MAX_KEYS) {
        // the keys in ascending order with d = value - must sum (ins / av hold the unsorted pairs meanwhile)
        const int32_t* p = d.payload + d.poff[r];
        const int32_t* kt = d.keys + d.key_off[s];
        for (int32_t j = lane; j < nt; j += 32) {
            const int32_t k = p[3 * j];
            const int32_t slot = (int32_t)d.key_off[s] + mono_col(kt, d.n_keys[s], k);
            W.ins[j] = k;
            W.av[j] = mono_join(p[3 * j + 1], p[3 * j + 2]) - rx_must(d, slot, iv);
        }
        __syncwarp();
        for (int32_t j = lane; j < nt; j += 32) {
            int32_t rank = 0;
            for (int32_t o = 0; o < nt; ++o) rank += W.ins[o] < W.ins[j];
            W.key[rank] = (int32_t)W.ins[j];
            W.d[rank] = W.av[j];
        }
        __syncwarp();
        // gather the "may" transfers; n > cap = too many
        auto find = [&](int64_t k) {
            int32_t a = 0, b = nt;
            while (a < b) {
                const int32_t c = (a + b) >> 1;
                if (W.key[c] < k) a = c + 1; else b = c;
            }
            return (int16_t)(a < nt && W.key[a] == k ? a : -1);
        };
        auto take = [&](bool valid, int32_t t) {
            int16_t jd = -1, jc = -1;
            if (valid) {
                const int32_t* q = d.t_rec + 3 * (int64_t)t;
                valid = !(d.t_M[t] < iv) && d.t_A[t] < cp && q[2] > 0;
                if (valid) {
                    jd = find(2 * (int64_t)q[0]);
                    jc = find(2 * (int64_t)q[1] + 1);
                    valid = jd >= 0 || jc >= 0;
                }
            }
            const unsigned bal = __ballot_sync(0xffffffffu, valid);
            const int32_t at = n + __popc(bal & ((1u << lane) - 1));
            if (valid && at < JTB_RX_MAX_GATHER) {
                W.cid[at] = d.t_id[t];
                W.ca[at] = d.t_rec[3 * (int64_t)t + 2];
                W.cjd[at] = jd;
                W.cjc[at] = jc;
            }
            n += __popc(bal);
        };
        const int32_t olo = d.ok_off[s], b = rx_lower(d.ok_inv, olo, d.ok_off[s + 1], cp);
        for (int32_t base = b - 1; base >= olo && n <= JTB_RX_MAX_GATHER; base -= 32) {
            const int32_t j = base - lane;
            const bool valid = j >= olo && d.ok_pmax[j] >= iv;
            if (!__any_sync(0xffffffffu, valid)) break;
            take(valid, valid ? d.ok_t[j] : 0);
        }
        const int32_t clo = d.cr_off[s], bc = rx_lower(d.cr_inv, clo, d.cr_off[s + 1], cp);
        for (int32_t base = clo; base < bc && n <= JTB_RX_MAX_GATHER; base += 32) {
            const int32_t j = base + lane;
            take(j < bc, j < bc ? d.cr_t[j] : 0);
        }
        __syncwarp();
        if (n <= JTB_RX_MAX_GATHER) {
            int32_t root_key;
            code = (int8_t)rx_search(W, nt, n, -1, d.max_nodes, lane, nodes, root_key, kept);
            if (code == JTB_RX_JOINT) {
                rkey = root_key;
                for (int32_t k = 0; k < nt; ++k) {
                    int32_t rk, kp;
                    if (rx_search(W, nt, n, k, d.max_nodes, lane, nodes, rk, kp) == JTB_RX_JOINT) {
                        code = JTB_RX_KEY;
                        rkey = W.key[k];
                        break;
                    }
                }
            }
        }
    }
    if (lane != 0) return;
    unsigned long long* c = d.cnt + (int64_t)s * 5;
    atomicAdd(&c[4], (unsigned long long)nodes);
    if (code == RX_EXPLAINED) { atomicAdd(&c[0], 1ull); return; }
    if (code == RX_UNDECIDED) { atomicAdd(&c[1], 1ull); return; }
    atomicAdd(&c[1 + code], 1ull);
    atomicMin(&d.wread[s], (unsigned long long)r);
    d.code[r] = code;
    d.rkey[r] = rkey;
    d.rmay[r] = kept;
    if (code == JTB_RX_KEY) {
        const int32_t* p = d.payload + d.poff[r];
        int64_t v = 0;
        for (int32_t j = 0; j < nt; ++j)
            if (p[3 * j] == rkey) v = mono_join(p[3 * j + 1], p[3 * j + 2]);
        const int32_t slot = (int32_t)d.key_off[s] + mono_col(d.keys + d.key_off[s], d.n_keys[s], rkey);
        d.rvalue[r] = v;
        d.rmust[r] = rx_must(d, slot, iv);
    }
}

// thread per transfer: is it must for its shard's witness read, on a key that read observes?
__global__ void rx_must_count(RxDev d) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= d.n_t) return;
    const int32_t s = d.t_shard[t];
    if (d.wread[s] == ~0ull) return;
    const int32_t r = (int32_t)d.wread[s];
    if (!(d.t_M[t] < d.r_inv[r])) return;
    const int32_t* q = d.t_rec + 3 * t;
    const int32_t* p = d.payload + d.poff[r];
    for (int32_t j = 0; j < d.ntrip[r]; ++j)
        if (p[3 * j] == 2 * q[0] || p[3 * j] == 2 * q[1] + 1) { atomicAdd(&d.nmust[s], 1); return; }
}

// ---- host ---------------------------------------------------------------------------------------------------------

inline int run_read_explanations(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                                 int64_t max_nodes, int32_t flags, jtb_rx_shard* shards, jtb_rx_result* out,
                                 std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    if (flags != 0) { err = "flags must be 0 (reserved)"; return -2; }
    if (int rc = check_history(h, false, err)) return rc;
    if (max_nodes <= 0) max_nodes = JTB_RX_DEFAULT_MAX_NODES;
    const int32_t S = h->n_shards;
    MonoHost H;
    if (int rc = mono_host_pass(h, H, err)) return rc;
    TlHost T;
    if (int rc = tl_host_pass(h, T, err)) return rc;
    if (T.t_id.size() > (size_t)1 << 30) { err = "more than 2^30 transfers"; return -2; }
    const int32_t m = (int32_t)H.r_shard.size(), nT = (int32_t)T.t_id.size(), nL = (int32_t)T.l_shard.size();
    const int64_t nR = T.rec_base.back();
    // the :ok and the crashed transfers of every shard, by invocation (the order of T)
    std::vector<int32_t> ok_t, ok_inv, ok_pmax, ok_off(S + 1, 0), cr_t, cr_inv, cr_off(S + 1, 0);
    for (int32_t s = 0; s < S; ++s) {
        int32_t run = INT_MIN;
        for (int32_t t = T.t_off[s]; t < T.t_off[s + 1]; ++t) {
            if (T.t_fate[t] == JTB_T_OK) {
                run = std::max(run, T.t_okcomp[t]);
                ok_t.push_back(t);
                ok_inv.push_back(T.t_inv[t]);
                ok_pmax.push_back(run);
            } else if (T.t_fate[t] != JTB_T_FAIL) {
                cr_t.push_back(t);
                cr_inv.push_back(T.t_inv[t]);
            }
        }
        ok_off[s + 1] = (int32_t)ok_t.size();
        cr_off[s + 1] = (int32_t)cr_t.size();
    }
    memset(out, 0, sizeof *out);
    for (int32_t s = 0; s < S; ++s) {
        jtb_rx_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_reads = H.n_reads[s];
        o.n_transfers = T.t_off[s + 1] - T.t_off[s];
        o.witness_index = o.key = -1;
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
    }
    float ms = 0;
    if (m > 0) {
        CallAllocs A;
        const int32_t slots = (int32_t)H.keys.size();
        TlDev d;
        RxDev x;
        d.n_t = x.n_t = nT;
        d.n_l = nL;
        d.n_rec = nR;
        x.m = m;
        x.n_c = 2 * nT;
        x.max_nodes = max_nodes;
        const int64_t* tid;
        TlTKey *tk0, *tk;
        TlRKey *rk0, *rk;
        int32_t *tid0, *tperm, *rv0, *rv, *tM, *tA, *nmust;
        uint64_t *mk, *ck0, *ck;
        int64_t *ca0, *ca, *cs;
        unsigned long long *cnt, *wread;
        uint8_t* tmp;
        JTB_OK(A.put(&d.payload, h->payload, (size_t)h->n_payload, st));
        x.payload = d.payload;
        JTB_OK(A.put(&x.poff, H.r_poff, st)); JTB_OK(A.put(&x.ntrip, H.r_ntrip, st)); JTB_OK(A.put(&x.r_shard, H.r_shard, st));
        JTB_OK(A.put(&x.r_inv, H.r_inv, st)); JTB_OK(A.put(&x.r_comp, H.r_comp, st));
        JTB_OK(A.put(&d.n_keys, H.n_keys, st)); JTB_OK(A.put(&d.key_off, H.key_off, st)); JTB_OK(A.put(&d.keys, H.keys, st));
        x.n_keys = d.n_keys; x.key_off = d.key_off; x.keys = d.keys;
        JTB_OK(A.put(&d.t_shard, T.t_shard, st)); JTB_OK(A.put(&tid, T.t_id, st)); JTB_OK(A.put(&d.t_rec, T.t_rec, st));
        JTB_OK(A.put(&d.t_inv, T.t_inv, st)); JTB_OK(A.put(&d.t_okcomp, T.t_okcomp, st));
        JTB_OK(A.put(&d.t_fate, T.t_fate, st)); JTB_OK(A.put(&d.t_off, T.t_off, st));
        x.t_shard = d.t_shard; x.t_rec = d.t_rec; x.t_id = tid;
        JTB_OK(A.put(&d.l_shard, T.l_shard, st)); JTB_OK(A.put(&d.l_comp, T.l_comp, st));
        JTB_OK(A.put(&d.l_poff, T.l_poff, st)); JTB_OK(A.put(&d.rec_base, T.rec_base, st));
        JTB_OK(A.put(&d.ib, T.ib, st)); JTB_OK(A.put(&d.ib_inv, T.ib_inv, st)); JTB_OK(A.put(&d.ib_off, T.ib_off, st));
        JTB_OK(A.put(&x.ok_t, ok_t, st)); JTB_OK(A.put(&x.ok_inv, ok_inv, st)); JTB_OK(A.put(&x.ok_pmax, ok_pmax, st));
        JTB_OK(A.put(&x.ok_off, ok_off, st)); JTB_OK(A.put(&x.cr_t, cr_t, st)); JTB_OK(A.put(&x.cr_inv, cr_inv, st));
        JTB_OK(A.put(&x.cr_off, cr_off, st));
        JTB_OK(A.alloc(&tk0, nT)); JTB_OK(A.alloc(&tk, nT)); JTB_OK(A.alloc(&tid0, nT)); JTB_OK(A.alloc(&tperm, nT));
        JTB_OK(A.alloc(&d.rec_slot, nR)); JTB_OK(A.alloc(&rk0, nR)); JTB_OK(A.alloc(&rk, nR));
        JTB_OK(A.alloc(&rv0, nR)); JTB_OK(A.alloc(&rv, nR));
        JTB_OK(A.alloc(&d.mlk, nT)); JTB_OK(A.alloc(&d.mv, nT)); JTB_OK(A.alloc(&d.mfrom, nT)); JTB_OK(A.alloc(&mk, nT));
        JTB_OK(A.alloc(&d.wid, (size_t)nL * 5)); JTB_OK(A.alloc(&d.count, (size_t)S * JTB_TL_KINDS));
        JTB_OK(A.alloc(&tM, nT)); JTB_OK(A.alloc(&tA, nT));
        JTB_OK(A.alloc(&ck0, 2 * (size_t)nT)); JTB_OK(A.alloc(&ck, 2 * (size_t)nT));
        JTB_OK(A.alloc(&ca0, 2 * (size_t)nT)); JTB_OK(A.alloc(&ca, 2 * (size_t)nT)); JTB_OK(A.alloc(&cs, 2 * (size_t)nT));
        JTB_OK(A.alloc(&x.code, m)); JTB_OK(A.alloc(&x.rkey, m)); JTB_OK(A.alloc(&x.rmay, m));
        JTB_OK(A.alloc(&x.rvalue, m)); JTB_OK(A.alloc(&x.rmust, m));
        JTB_OK(A.alloc(&cnt, (size_t)S * 5)); JTB_OK(A.alloc(&wread, S)); JTB_OK(A.alloc(&nmust, S));
        d.tkey = tk; d.tperm = tperm; d.rkey = rk; d.rval = rv;
        x.t_M = tM; x.t_A = tA; x.ckey = ck; x.csum = cs; x.cnt = cnt; x.wread = wread; x.nmust = nmust;
        size_t tmp_t = 0, tmp_r = 0, tmp_c = 0, tmp_s = 0;
        if (nT > 0) {
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_t, tk0, tk, tid0, tperm, nT, TlTKeyDecomposer{}, st));
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_c, ck0, ck, ca0, ca, 2 * nT, 0, 64, st));
            JTB_OK(cub::DeviceScan::InclusiveSumByKey(nullptr, tmp_s, (const uint64_t*)ck, (const int64_t*)ca, cs,
                                                      2 * nT, CbSlotEq{}, st));
        }
        if (nR > 0)
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_r, rk0, rk, rv0, rv, (int)nR, TlRKeyDecomposer{}, st));
        const size_t tmp_bytes = std::max({tmp_t, tmp_r, tmp_c, tmp_s});
        JTB_OK(A.alloc(&tmp, tmp_bytes));
        auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };

        JTB_OK(cudaEventRecord(ev0, st));
        JTB_OK(cudaMemsetAsync(d.mlk, 0x7f, (size_t)nT * 4, st));   // 0x7f7f7f7f > any lookup id: "none"
        JTB_OK(cudaMemsetAsync(d.wid, 0xff, (size_t)nL * 40, st));
        JTB_OK(cudaMemsetAsync(d.count, 0, (size_t)S * JTB_TL_KINDS * 8, st));
        JTB_OK(cudaMemsetAsync(cnt, 0, (size_t)S * 40, st));
        JTB_OK(cudaMemsetAsync(wread, 0xff, (size_t)S * 8, st));
        JTB_OK(cudaMemsetAsync(nmust, 0, (size_t)S * 4, st));
        size_t tb;
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
            rx_contrib<<<grid(nT, 256), 256, 0, st>>>(d, slots, tM, ck0, ca0);
            tb = tmp_bytes;
            JTB_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, ck0, ck, ca0, ca, 2 * nT, 0, 64, st));
            tb = tmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveSumByKey(tmp, tb, (const uint64_t*)ck, (const int64_t*)ca, cs, 2 * nT,
                                                      CbSlotEq{}, st));
        }
        rx_reads<<<grid(m, RX_WARPS), RX_WARPS * 32, 0, st>>>(x);
        if (nT > 0) rx_must_count<<<grid(nT, 256), 256, 0, st>>>(x);
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<unsigned long long> cnt_h((size_t)S * 5), wread_h(S);
        std::vector<int32_t> nmust_h(S);
        JTB_OK(cudaMemcpyAsync(cnt_h.data(), cnt, cnt_h.size() * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(wread_h.data(), wread, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(nmust_h.data(), nmust, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        for (int32_t s = 0; s < S; ++s) {
            jtb_rx_shard& o = shards[s];
            const unsigned long long* c = &cnt_h[(size_t)s * 5];
            o.n_explained = (int64_t)c[0];
            o.n_undecided = (int64_t)c[1];
            o.count_by_kind[0] = (int64_t)c[2];
            o.count_by_kind[1] = (int64_t)c[3];
            o.nodes = (int64_t)c[4];
            if (wread_h[s] != ~0ull) {   // the witness read's fields: a few scalars of one read per INVALID shard
                const int32_t r = (int32_t)wread_h[s];
                int8_t code;
                JTB_OK(cudaMemcpy(&code, x.code + r, 1, cudaMemcpyDeviceToHost));
                JTB_OK(cudaMemcpy(&o.key, x.rkey + r, 4, cudaMemcpyDeviceToHost));
                JTB_OK(cudaMemcpy(&o.n_may, x.rmay + r, 4, cudaMemcpyDeviceToHost));
                o.kind = code;
                o.witness_index = h->index[H.r_ev[r]];
                o.n_must = nmust_h[s];
                if (code == JTB_RX_KEY) {
                    JTB_OK(cudaMemcpy(&o.value, x.rvalue + r, 8, cudaMemcpyDeviceToHost));
                    JTB_OK(cudaMemcpy(&o.must_sum, x.rmust + r, 8, cudaMemcpyDeviceToHost));
                }
                o.valid = JTB_INVALID;
            } else if (o.n_undecided > 0) {
                o.valid = JTB_UNKNOWN;
            }
            out->n_explained += o.n_explained;
            out->n_unexplained += o.count_by_kind[0] + o.count_by_kind[1];
            out->n_undecided += o.n_undecided;
            out->nodes += o.nodes;
        }
    }
    roll_up(out, shards, S, ms, t0);
    return 0;
}

}  // namespace jtb
