// jtb_counter_bounds.cuh — K8: the counter-bounds check (every ledger read held to the transfers around it) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K8 counter-bounds check"): every key k an :ok read r observes must lie in
// [L_k(r), U_k(r)], L = the :ok transfers on k completed before r's invocation, U = the non-:fail transfers on k invoked
// before r's completion.  The reads, their invocations and the shards' key tables are K7's host pass (mono_host_pass);
// this file adds transfer pairing and one contribution record per (transfer, observed key), slot = the key's index in
// the concatenated key tables.  On the device: two cub radix sorts of the contributions, by (slot, completion position)
// (the L list; a transfer that is not :ok has completion INT_MAX and so sorts after every :ok one of its slot and is
// never counted) and by (slot, invocation position) (the U list), a cub inclusive sum by slot of the amounts of each,
// then a warp per read, a lane per triple, two binary searches per triple.  A thread per INVALID shard explains it.
#pragma once
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "../../include/jtb_check.h"
#include "jtb_call.cuh"
#include "jtb_monotonic.cuh"

namespace jtb {

// the device's view of one call.  keyL / keyU: the sorted 64-bit keys (slot << 32 | position); idL / idU: contribution
// ids in that order; sumL / sumU: inclusive prefix sums of the amounts per slot in that order.  Both lists have the same
// slot segments [off[slot], off[slot + 1]).
struct CbDev {
    int32_t m = 0;                          // reads
    const int32_t* payload = nullptr;
    const int64_t* poff = nullptr;          // [m]
    const int32_t* ntrip = nullptr;         // [m]
    const int32_t* shard = nullptr;         // [m]
    const int32_t* inv = nullptr;           // [m] invocation position, -1 = none
    const int32_t* comp = nullptr;          // [m] completion position
    const int32_t* n_keys = nullptr;        // [n_shards]
    const int64_t* key_off = nullptr;       // [n_shards + 1] into keys (= the shard's first slot)
    const int32_t* keys = nullptr;          // per shard, ascending
    const int32_t* off = nullptr;           // [slots + 1] contribution segments
    const uint64_t* keyL = nullptr;
    const uint64_t* keyU = nullptr;
    const int32_t* idL = nullptr;
    const int32_t* idU = nullptr;
    const int64_t* sumL = nullptr;
    const int64_t* sumU = nullptr;
};

struct CbSlotEq {
    __host__ __device__ bool operator()(uint64_t a, uint64_t b) const { return (a >> 32) == (b >> 32); }
};

// first j in [lo, hi) with key[j] > x (keys ascending)
__device__ __forceinline__ int32_t cb_upper(const uint64_t* __restrict__ key, int32_t lo, int32_t hi, uint64_t x) {
    while (lo < hi) {
        const int32_t c = (int32_t)(((int64_t)lo + hi) >> 1);
        if (key[c] <= x) lo = c + 1; else hi = c;
    }
    return lo;
}

// the two bounds of read r on slot `slot`: jl / ju = the end of the counted prefix of the L / U list
__device__ __forceinline__ void cb_bounds(const CbDev& d, int32_t r, int32_t slot, int64_t& L, int64_t& U, int32_t& jl,
                                          int32_t& ju) {
    const int32_t lo = d.off[slot], hi = d.off[slot + 1];
    const uint64_t base = (uint64_t)(uint32_t)slot << 32;
    const int32_t iv = d.inv[r];
    jl = iv < 0 ? lo : cb_upper(d.keyL, lo, hi, base | (uint32_t)iv);
    ju = cb_upper(d.keyU, lo, hi, base | (uint32_t)d.comp[r]);
    L = jl > lo ? d.sumL[jl - 1] : 0;
    U = ju > lo ? d.sumU[ju - 1] : 0;
}

// thread per contribution: both sort keys (completion INT_MAX for transfers that are not :ok)
__global__ void cb_keys(int32_t n, const int32_t* __restrict__ slot, const int32_t* __restrict__ inv,
                        const int32_t* __restrict__ comp, uint64_t* __restrict__ keyL, uint64_t* __restrict__ keyU,
                        int32_t* __restrict__ ids) {
    const int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (c >= n) return;
    const uint64_t base = (uint64_t)(uint32_t)slot[c] << 32;
    keyL[c] = base | (uint32_t)comp[c];
    keyU[c] = base | (uint32_t)inv[c];
    ids[c] = (int32_t)c;
}

// thread per sorted position: the amounts in L order and in U order
__global__ void cb_gather(int32_t n, const int32_t* __restrict__ amount, const int32_t* __restrict__ idL,
                          const int32_t* __restrict__ idU, int64_t* __restrict__ aL, int64_t* __restrict__ aU) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n) return;
    aL[j] = amount[idL[j]];
    aU[j] = amount[idU[j]];
}

// warp per read, lane per (key, value) triple: compare the value with [L, U]; per shard count the violations of each
// kind and keep the earliest (read id, column).  Read ids ascend with the completion position inside a shard, so the
// smallest read id is the earliest completion.
__global__ void cb_check(CbDev d, unsigned long long* __restrict__ n_below, unsigned long long* __restrict__ n_above,
                         unsigned long long* __restrict__ wkey) {
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= d.m) return;
    const int32_t r = (int32_t)w, sh = d.shard[r], K = d.n_keys[sh], nt = d.ntrip[r];
    const int32_t* kt = d.keys + d.key_off[sh];
    const int32_t* p = d.payload + d.poff[r];
    unsigned below = 0, above = 0;
    int32_t first = INT_MAX;
    for (int32_t j = lane; j < nt; j += 32) {
        const int32_t a = mono_col(kt, K, p[3 * j]);   // the host pass put every observed key in the table
        const int64_t v = mono_join(p[3 * j + 1], p[3 * j + 2]);
        int64_t L, U;
        int32_t jl, ju;
        cb_bounds(d, r, (int32_t)d.key_off[sh] + a, L, U, jl, ju);
        const bool lo = v < L, hi = v > U;
        below += lo;
        above += hi;
        if (lo || hi) first = min(first, a);
    }
    for (int o = 16; o; o >>= 1) {
        below += __shfl_down_sync(0xffffffffu, below, o);
        above += __shfl_down_sync(0xffffffffu, above, o);
        first = min(first, __shfl_down_sync(0xffffffffu, first, o));
    }
    if (lane == 0 && (below || above)) {
        if (below) atomicAdd(&n_below[sh], (unsigned long long)below);
        if (above) atomicAdd(&n_above[sh], (unsigned long long)above);
        atomicMin(&wkey[sh], (unsigned long long)(uint32_t)r << 32 | (uint32_t)first);
    }
}

struct CbWitness {
    int32_t read, key, kind, culprit;
    int64_t value, bound;
};

// thread per shard with a witness: its read, key, kind, value, bound and culprit
__global__ void cb_explain(CbDev d, int32_t n_shards, const unsigned long long* __restrict__ wkey,
                           const int32_t* __restrict__ c_cidx, const int32_t* __restrict__ c_iidx,
                           CbWitness* __restrict__ out) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_shards || wkey[s] == ~0ull) return;
    const int32_t r = (int32_t)(wkey[s] >> 32), col = (int32_t)(wkey[s] & 0xffffffffu);
    const int32_t slot = (int32_t)d.key_off[s] + col, key = d.keys[slot];
    const int32_t* p = d.payload + d.poff[r];
    int64_t v = 0;
    for (int32_t j = 0; j < d.ntrip[r]; ++j)
        if (p[3 * j] == key) { v = mono_join(p[3 * j + 1], p[3 * j + 2]); break; }
    int64_t L, U;
    int32_t jl, ju;
    cb_bounds(d, r, slot, L, U, jl, ju);
    CbWitness o{r, key, 0, -1, v, 0};
    const int32_t lo = d.off[slot];
    if (v < L) {
        // the first position of the L list whose running sum exceeds v (v < L = sumL[jl - 1], so one exists); a
        // negative value below an empty L has none
        int32_t a = lo, b = jl - 1;
        while (a < b) {
            const int32_t c = (a + b) >> 1;
            if (d.sumL[c] > v) b = c; else a = c + 1;
        }
        o.kind = JTB_CB_BELOW;
        o.bound = L;
        o.culprit = jl > lo ? c_cidx[d.idL[a]] : -1;
    } else {
        o.kind = JTB_CB_ABOVE;
        o.bound = U;
        o.culprit = ju > lo ? c_iidx[d.idU[ju - 1]] : -1;
    }
    out[s] = o;
}

// ---- host ---------------------------------------------------------------------------------------------------------

// One contribution per (transfer, key of its shard's table): the transfer adds `amount` to that key.
struct CbContrib {
    std::vector<int32_t> slot, inv, comp, amount, iidx, cidx;   // comp = INT_MAX, cidx = -1 unless :ok
    std::vector<int32_t> n_transfers;                           // [n_shards] non-:fail transfers
    std::vector<int32_t> off;                                   // [slots + 1]
};

// Pair every transfer invoke with the next event of its process, validate it, and emit its contributions to the keys
// the shard's :ok reads observe.  Shards must already be CSR-checked (mono_host_pass does).
inline int cb_transfer_pass(const jtb_history* h, const MonoHost& H, CbContrib& C, std::string& err) {
    const int32_t S = h->n_shards;
    C.n_transfers.assign(S, 0);
    std::vector<int64_t> cnt(H.keys.size() + 1, 0);
    std::unordered_map<int32_t, int64_t> open;   // process -> event of its pending transfer invoke
    for (int32_t s = 0; s < S; ++s) {
        const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
        const int32_t* kt = H.keys.data() + H.key_off[s];
        const int32_t K = H.n_keys[s];
        open.clear();
        auto resolve = [&](int64_t ie, int64_t ce) -> int {   // ce = the fate event, -1 = never completed
            const int32_t fate = ce < 0 ? -1 : h->type[ce];
            if (fate == JTB_T_FAIL) return 0;
            C.n_transfers[s]++;
            const int32_t acct[2] = {h->b[ie], h->c[ie]};
            for (int field = 0; field < 2; ++field) {
                const int32_t key = 2 * acct[field] + field;
                const int32_t col = mono_col(kt, K, key);
                if (col == K || kt[col] != key) continue;   // no :ok read of the shard observes it
                if (C.slot.size() >= (size_t)INT_MAX) { err = "more than 2^31-1 transfer contributions"; return -2; }
                const int32_t slot = (int32_t)H.key_off[s] + col;
                const bool ok = fate == JTB_T_OK;
                C.slot.push_back(slot);
                C.inv.push_back((int32_t)(ie - lo));
                C.comp.push_back(ok ? (int32_t)(ce - lo) : INT_MAX);
                C.amount.push_back(h->a[ie]);
                C.iidx.push_back(h->index[ie]);
                C.cidx.push_back(ok ? h->index[ce] : -1);
                cnt[slot + 1]++;
            }
            return 0;
        };
        for (int64_t e = lo; e < hi; ++e) {
            const int32_t p = h->process[e];
            if (p < 0) continue;
            auto it = open.find(p);
            if (it != open.end()) {
                const int64_t ie = it->second;
                open.erase(it);
                if (int rc = resolve(ie, h->type[e] == JTB_T_INVOKE ? -1 : e)) return rc;
            }
            if (h->type[e] != JTB_T_INVOKE || h->f[e] != JTB_F_TRANSFER) continue;
            if (h->a[e] < 0) return input_error(err, "transfer at :index %d: negative amount %d", h->index[e], h->a[e]);
            if (h->b[e] < 0 || h->b[e] >= (1 << 30) || h->c[e] < 0 || h->c[e] >= (1 << 30))
                return input_error(err, "transfer at :index %d: account outside [0, 2^30)", h->index[e]);
            open.emplace(p, e);
        }
        // never completed, in invocation order (the order only decides the record order, which the sorts erase)
        std::vector<int64_t> rest;
        for (auto& [p, ie] : open) rest.push_back(ie);
        std::sort(rest.begin(), rest.end());
        for (int64_t ie : rest)
            if (int rc = resolve(ie, -1)) return rc;
    }
    C.off.resize(cnt.size());
    for (size_t i = 0; i < cnt.size(); ++i) C.off[i] = (int32_t)(cnt[i] + (i ? C.off[i - 1] : 0));
    return 0;
}

inline int run_counter_bounds(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, int32_t flags,
                              jtb_cb_shard* shards, jtb_cb_result* out, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    if (flags != 0) { err = "flags must be 0 (reserved)"; return -2; }
    if (int rc = check_history(h, true, err)) return rc;
    const int32_t S = h->n_shards;
    MonoHost H;
    if (int rc = mono_host_pass(h, H, err)) return rc;
    CbContrib C;
    if (int rc = cb_transfer_pass(h, H, C, err)) return rc;
    memset(out, 0, sizeof *out);
    for (int32_t s = 0; s < S; ++s) {
        jtb_cb_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_reads = H.n_reads[s];
        o.n_transfers = C.n_transfers[s];
        o.n_keys = H.n_keys[s];
        o.witness_index = o.witness_key = o.culprit_index = -1;
        out->n_reads += H.n_reads[s];
        out->n_transfers += C.n_transfers[s];
    }
    const int32_t m = (int32_t)H.r_shard.size(), n = (int32_t)C.slot.size();
    float ms = 0;
    if (m > 0) {
        CallAllocs A;
        CbDev d;
        d.m = m;
        const size_t slots = H.keys.size();
        const int32_t *cslot, *cinv, *ccomp, *camt, *ciidx, *ccidx;
        uint64_t *k0, *k1, *kL, *kU;
        int32_t *id0, *idL, *idU;
        int64_t *aL, *aU, *sL, *sU;
        unsigned long long *below, *above, *wkey;
        CbWitness* wit;
        uint8_t* tmp;
        JTB_OK(A.put(&d.payload, h->payload, (size_t)h->n_payload, st));
        JTB_OK(A.put(&d.poff, H.r_poff, st)); JTB_OK(A.put(&d.ntrip, H.r_ntrip, st)); JTB_OK(A.put(&d.shard, H.r_shard, st));
        JTB_OK(A.put(&d.inv, H.r_inv, st)); JTB_OK(A.put(&d.comp, H.r_comp, st));
        JTB_OK(A.put(&d.n_keys, H.n_keys, st)); JTB_OK(A.put(&d.key_off, H.key_off, st)); JTB_OK(A.put(&d.keys, H.keys, st));
        JTB_OK(A.put(&d.off, C.off, st));
        JTB_OK(A.put(&cslot, C.slot, st)); JTB_OK(A.put(&cinv, C.inv, st)); JTB_OK(A.put(&ccomp, C.comp, st));
        JTB_OK(A.put(&camt, C.amount, st)); JTB_OK(A.put(&ciidx, C.iidx, st)); JTB_OK(A.put(&ccidx, C.cidx, st));
        JTB_OK(A.alloc(&k0, n)); JTB_OK(A.alloc(&k1, n));
        JTB_OK(A.alloc(&kL, n)); JTB_OK(A.alloc(&kU, n));
        JTB_OK(A.alloc(&id0, n)); JTB_OK(A.alloc(&idL, n)); JTB_OK(A.alloc(&idU, n));
        JTB_OK(A.alloc(&aL, n)); JTB_OK(A.alloc(&aU, n));
        JTB_OK(A.alloc(&sL, n)); JTB_OK(A.alloc(&sU, n));
        JTB_OK(A.alloc(&below, S)); JTB_OK(A.alloc(&above, S)); JTB_OK(A.alloc(&wkey, S));
        JTB_OK(A.alloc(&wit, S));
        d.keyL = kL; d.keyU = kU;
        d.idL = idL; d.idU = idU;
        d.sumL = sL; d.sumU = sU;
        // keys = slot << 32 | position: the bits above the largest slot are zero
        int end_bit = 32;
        while (end_bit < 64 && (slots >> (end_bit - 32)) != 0) ++end_bit;
        size_t tmp_sort = 0, tmp_scan = 0;
        if (n > 0) {
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, k0, kL, id0, idL, n, 0, end_bit, st));
            JTB_OK(cub::DeviceScan::InclusiveSumByKey(nullptr, tmp_scan, d.keyL, (const int64_t*)aL, sL, n, CbSlotEq{},
                                                      st));
        }
        const size_t tmp_bytes = std::max(tmp_sort, tmp_scan);
        JTB_OK(A.alloc(&tmp, tmp_bytes));
        const unsigned c_grid = (unsigned)(((int64_t)n + 255) / 256);
        const unsigned warp_grid = (unsigned)(((int64_t)m * 32 + 255) / 256);
        const unsigned sh_grid = (unsigned)((S + 255) / 256);

        JTB_OK(cudaEventRecord(ev0, st));
        JTB_OK(cudaMemsetAsync(below, 0, (size_t)S * 8, st));
        JTB_OK(cudaMemsetAsync(above, 0, (size_t)S * 8, st));
        JTB_OK(cudaMemsetAsync(wkey, 0xff, (size_t)S * 8, st));
        if (n > 0) {
            cb_keys<<<c_grid, 256, 0, st>>>(n, cslot, cinv, ccomp, k0, k1, id0);
            size_t tb = tmp_bytes;
            JTB_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, k0, kL, id0, idL, n, 0, end_bit, st));
            tb = tmp_bytes;
            JTB_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, k1, kU, id0, idU, n, 0, end_bit, st));
            cb_gather<<<c_grid, 256, 0, st>>>(n, camt, d.idL, d.idU, aL, aU);
            tb = tmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveSumByKey(tmp, tb, d.keyL, (const int64_t*)aL, sL, n, CbSlotEq{}, st));
            tb = tmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveSumByKey(tmp, tb, d.keyU, (const int64_t*)aU, sU, n, CbSlotEq{}, st));
        }
        cb_check<<<warp_grid, 256, 0, st>>>(d, below, above, wkey);
        cb_explain<<<sh_grid, 256, 0, st>>>(d, S, wkey, ccidx, ciidx, wit);
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<unsigned long long> below_h(S), above_h(S), wkey_h(S);
        std::vector<CbWitness> wit_h(S);
        JTB_OK(cudaMemcpyAsync(below_h.data(), below, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(above_h.data(), above, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(wkey_h.data(), wkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(wit_h.data(), wit, (size_t)S * sizeof(CbWitness), cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        for (int32_t s = 0; s < S; ++s) {
            jtb_cb_shard& o = shards[s];
            o.n_below = (int64_t)below_h[s];
            o.n_above = (int64_t)above_h[s];
            out->n_violations += o.n_below + o.n_above;
            if (wkey_h[s] == ~0ull) continue;
            const CbWitness& w = wit_h[s];
            o.valid = JTB_INVALID;
            o.witness_index = h->index[H.r_ev[w.read]];
            o.witness_key = w.key;
            o.kind = w.kind;
            o.culprit_index = w.culprit;
            o.value = w.value;
            o.bound = w.bound;
        }
    }
    roll_up(out, shards, S, ms, t0);
    return 0;
}

}  // namespace jtb
