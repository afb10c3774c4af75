// jtb_monotonic.cuh — K7: the monotonic-key check (Elle's monotonic-key graph plus real-time order) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K7 monotonic-key check"): the :ok reads of a shard are the nodes; r -> s
// when r observed a strictly smaller value than s for some key, or (real time) r completed before s was invoked.  On
// a shard whose reads all observe the same key set the graph has a cycle iff it has a 2-cycle, and sorting the reads
// by (S = sum of the values, invocation position) turns the decision into two linear passes:
//   (a) some key's value decreases between two ADJACENT reads of that order, or
//   (b) some read has a read later in the order that completed before it was invoked (segmented suffix-min).
// Layout: a read-major dense matrix V[read][column] (int64, columns = the shard's keys in ascending order), one
// stable radix sort of (shard, S as 128 bits, invocation) with cub, one segmented scan, a warp per adjacent pair.
// The witness is a binary search over the completion-position bound (all INVALID shards at once, the same decision
// on the masked prefix), the partner a scan of the reads for a 2-cycle with the witness read.
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
#include <cuda/std/tuple>
#include <cuda_runtime.h>

#include "../../include/jtb_check.h"
#include "jtb_call.cuh"

namespace jtb {

struct MonoKey {
    uint32_t shard;
    uint32_t inv;   // invocation position + 1 (0 = no invocation seen)
    uint64_t hi;    // S as a signed 128-bit number, sign bit flipped so that unsigned order is signed order
    uint64_t lo;
};
struct MonoKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, uint64_t&, uint64_t&, uint32_t&> operator()(MonoKey& k) const {
        return {k.shard, k.hi, k.lo, k.inv};
    }
};

// one element of the reversed, segmented suffix-min scan: the smallest completion position and the smallest sorted
// position among the SELECTED reads at or after a position of the sort, within one shard
struct MonoSuffix {
    int32_t shard, comp, pos;
};
struct MonoSuffixMin {
    __host__ __device__ MonoSuffix operator()(const MonoSuffix& a, const MonoSuffix& b) const {
        if (a.shard != b.shard) return b;   // shards are contiguous in the sort: a new shard restarts the scan
        return {b.shard, min(a.comp, b.comp), min(a.pos, b.pos)};
    }
};

struct MonoDev {
    int32_t m = 0;                      // reads on the device
    const int32_t* shard = nullptr;     // [m] shard of each read
    const int32_t* inv = nullptr;       // [m] invocation position in its shard, -1 = none
    const int32_t* comp = nullptr;      // [m] completion position in its shard
    const int64_t* row = nullptr;       // [m] offset of the read's row in V
    const int32_t* n_keys = nullptr;    // [n_shards] row width
    const int32_t* ord = nullptr;       // [m] read ids in sort order
    const int64_t* V = nullptr;
};

// A shard's key table (MonoHost::keys, kt[0, K), ascending): the column of key, i.e. the first c with kt[c] >= key
__host__ __device__ __forceinline__ int32_t mono_col(const int32_t* kt, int32_t K, int32_t key) {
    int32_t a = 0, b = K;
    while (a < b) {
        const int32_t c = (a + b) >> 1;
        if (kt[c] < key) a = c + 1; else b = c;
    }
    return a;
}

// the int64 a payload stores as two int32 words, the low word first
__host__ __device__ __forceinline__ int64_t mono_join(int32_t lo, int32_t hi) {
    return (int64_t)(((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo);
}

__device__ __forceinline__ void mono_add128(uint64_t& lo, uint64_t& hi, uint64_t blo, uint64_t bhi) {
    const uint64_t l = lo + blo;
    hi = hi + bhi + (l < lo ? 1ull : 0ull);
    lo = l;
}

// warp per read: scatter its (key, value) triples into its row of V (column = rank of the key among the shard's
// keys) and write its sort key (shard, S, invocation)
__global__ void mono_scatter(int32_t m, const int32_t* __restrict__ payload, const int64_t* __restrict__ poff,
                             const int32_t* __restrict__ shard, const int32_t* __restrict__ inv,
                             const int64_t* __restrict__ row, const int32_t* __restrict__ n_keys,
                             const int64_t* __restrict__ key_off, const int32_t* __restrict__ keys,
                             int64_t* __restrict__ V, MonoKey* __restrict__ sort_key, int32_t* __restrict__ ids) {
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= m) return;
    const int32_t r = (int32_t)w, sh = shard[r], K = n_keys[sh];
    const int32_t* kt = keys + key_off[sh];
    const int32_t* p = payload + poff[r];
    int64_t* vr = V + row[r];
    uint64_t lo = 0, hi = 0;
    for (int32_t j = lane; j < K; j += 32) {
        const int32_t key = p[3 * j];
        const int64_t v = mono_join(p[3 * j + 1], p[3 * j + 2]);
        vr[mono_col(kt, K, key)] = v;   // the host checked that every key is in the table
        mono_add128(lo, hi, (uint64_t)v, v < 0 ? ~0ull : 0ull);
    }
    for (int o = 16; o; o >>= 1) {
        const uint64_t olo = __shfl_down_sync(0xffffffffu, lo, o), ohi = __shfl_down_sync(0xffffffffu, hi, o);
        mono_add128(lo, hi, olo, ohi);
    }
    if (lane == 0) {
        sort_key[r] = MonoKey{(uint32_t)sh, (uint32_t)(inv[r] + 1), hi ^ 0x8000000000000000ull, lo};
        ids[r] = r;
    }
}

// the scan input, reversed: element j describes sorted position m-1-j (a read is selected when its completion
// position is <= bound[shard]; INT_MAX stands for "none")
__global__ void mono_suffix_init(MonoDev d, const int32_t* __restrict__ bound, MonoSuffix* __restrict__ rev) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= d.m) return;
    const int32_t i = d.m - 1 - (int32_t)j, r = d.ord[i], sh = d.shard[r];
    const bool sel = d.comp[r] <= bound[sh];
    rev[j] = MonoSuffix{sh, sel ? d.comp[r] : INT_MAX, sel ? i : INT_MAX};
}

// warp per sorted position i of a selected read r: q = the next selected read of the shard in the order.
// (a) a column with V[r] > V[q];  (b) a later selected read completed before r was invoked.
__global__ void mono_check(MonoDev d, const int32_t* __restrict__ bound, const MonoSuffix* __restrict__ scan,
                           int realtime, int32_t* __restrict__ bad) {
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= d.m - 1) return;   // the last position has no successor
    const int32_t i = (int32_t)w, r = d.ord[i], sh = d.shard[r];
    if (d.comp[r] > bound[sh]) return;
    const MonoSuffix nx = scan[d.m - 2 - i];   // suffix over sorted positions >= i + 1
    if (nx.shard != sh || nx.pos == INT_MAX) return;
    bool v = realtime && nx.comp < d.inv[r];
    if (!v) {
        const int32_t q = d.ord[nx.pos], K = d.n_keys[sh];
        const int64_t* a = d.V + d.row[r];
        const int64_t* b = d.V + d.row[q];
        bool dec = false;
        for (int32_t c = lane; c < K; c += 32) dec |= a[c] > b[c];
        v = __any_sync(0xffffffffu, dec);
    }
    if (v && lane == 0) atomicOr(&bad[sh], 1);
}

// verdict pass: every read of a searched shard selected
__global__ void mono_bound_all(int32_t n, int32_t* __restrict__ bound, int32_t* __restrict__ bad) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) { bound[s] = INT_MAX; bad[s] = 0; }
}

// witness search, one step per INVALID shard: test the prefix of completions <= mid
__global__ void mono_bound_mid(int32_t n, const int32_t* __restrict__ lo, const int32_t* __restrict__ hi,
                               int32_t* __restrict__ bound, int32_t* __restrict__ bad) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    bound[s] = lo[s] < hi[s] ? (int32_t)(((int64_t)lo[s] + hi[s]) >> 1) : -1;
    bad[s] = 0;
}

__global__ void mono_bound_update(int32_t n, int32_t* __restrict__ lo, int32_t* __restrict__ hi,
                                  const int32_t* __restrict__ bound, const int32_t* __restrict__ bad) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || lo[s] >= hi[s]) return;
    if (bad[s]) hi[s] = bound[s]; else lo[s] = bound[s] + 1;
}

// the witness read of an INVALID shard: the read completing at the bound the search converged to (wpos = -1 for
// shards that are not searched)
__global__ void mono_find_witness(MonoDev d, const int32_t* __restrict__ wpos, int32_t* __restrict__ wit) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= d.m) return;
    const int32_t sh = d.shard[r];
    if (wpos[sh] >= 0 && d.comp[r] == wpos[sh]) wit[sh] = (int32_t)r;
}

// thread per read r of the witness' prefix: does r form a 2-cycle with the witness read s?  The smallest completion
// :index wins (key = biased :index << 32 | read id)
__global__ void mono_partner(MonoDev d, const int32_t* __restrict__ wpos, const int32_t* __restrict__ wit,
                             const int32_t* __restrict__ cidx, int realtime, unsigned long long* __restrict__ pkey) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= d.m) return;
    const int32_t r = (int32_t)t, sh = d.shard[r];
    if (wpos[sh] < 0 || d.comp[r] > wpos[sh]) return;
    const int32_t s = wit[sh];
    if (s == r) return;
    const int32_t K = d.n_keys[sh];
    const int64_t* a = d.V + d.row[r];
    const int64_t* b = d.V + d.row[s];
    bool up = false, down = false;
    for (int32_t c = 0; c < K; ++c) { up |= a[c] < b[c]; down |= a[c] > b[c]; }
    const bool rs = up || (realtime && d.comp[r] < d.inv[s]);
    const bool sr = down || (realtime && d.comp[s] < d.inv[r]);
    if (rs && sr) atomicMin(&pkey[sh], (unsigned long long)((uint32_t)cidx[r] ^ 0x80000000u) << 32 | (uint32_t)r);
}

// ---- host ---------------------------------------------------------------------------------------------------------

// The host pass: pair every :ok read with its invocation, validate its payload, give every shard its sorted key table
// and find the shards with partial reads.  Reads of one shard are contiguous and in history order.
struct MonoHost {
    std::vector<int32_t> r_shard, r_inv, r_comp, r_ntrip;
    std::vector<int64_t> r_ev, r_poff;
    std::vector<int32_t> n_reads, n_keys, min_trip;
    std::vector<int64_t> key_off;   // [n_shards + 1] into keys
    std::vector<int32_t> keys;      // per shard, ascending
};

inline int mono_host_pass(const jtb_history* h, MonoHost& H, std::string& err) {
    const int32_t S = h->n_shards;
    H.n_reads.assign(S, 0);
    H.n_keys.assign(S, 0);
    H.min_trip.assign(S, INT_MAX);
    H.key_off.assign((size_t)S + 1, 0);
    int32_t max_proc = -1;
    for (int64_t e = 0; e < h->n_events; ++e) max_proc = std::max(max_proc, h->process[e]);
    // last invoke of each process: (shard stamp, position); a direct table unless the process ids are huge
    const bool direct = max_proc < (1 << 24);
    std::vector<int64_t> last(direct ? (size_t)max_proc + 1 : 0, -1);
    std::unordered_map<int32_t, int64_t> last_map;
    std::unordered_map<int32_t, int32_t> col_of;
    std::vector<int32_t> prov, hint, seen;
    for (int32_t s = 0; s < S; ++s) {
        const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
        if (lo < 0 || hi < lo || hi > h->n_events) { err = "shard_off is not a CSR partition of the events"; return -2; }
        if (hi - lo > INT_MAX) { err = "a shard has more than 2^31-1 events"; return -2; }
        col_of.clear();
        prov.clear();
        hint.clear();
        if (!direct) last_map.clear();
        for (int64_t e = lo; e < hi; ++e) {
            const int32_t p = h->process[e];
            if (p < 0) continue;
            const int32_t pos = (int32_t)(e - lo);
            const int64_t stamp = ((int64_t)s << 32) | (uint32_t)pos;
            if (h->type[e] == JTB_T_INVOKE) {
                if (direct) last[p] = stamp; else last_map[p] = stamp;
                continue;
            }
            if (h->type[e] != JTB_T_OK || h->f[e] != JTB_F_READ || h->payload_len[e] < 0) continue;
            int64_t li = -1;
            if (direct) li = last[p];
            else { auto it = last_map.find(p); if (it != last_map.end()) li = it->second; }
            const int32_t inv = (li >= 0 && (li >> 32) == s) ? (int32_t)(li & 0xffffffff) : -1;
            const int32_t len = h->payload_len[e];
            const int64_t off = h->payload_off[e];
            if (len % 3 != 0)
                return input_error(err, "read at :index %d: payload length %d is not a multiple of 3", h->index[e], len);
            if (off < 0 || off + len > h->n_payload)
                return input_error(err, "read at :index %d: payload out of range", h->index[e]);
            if (H.r_shard.size() >= (size_t)INT_MAX) { err = "more than 2^31-1 reads"; return -2; }
            const int32_t rid = (int32_t)H.r_shard.size(), nt = len / 3;
            const int32_t* p3 = h->payload + off;
            for (int32_t j = 0; j < nt; ++j) {
                const int32_t key = p3[3 * j];
                int32_t col;
                if (j < (int32_t)hint.size() && prov[hint[j]] == key) col = hint[j];
                else {
                    auto it = col_of.find(key);
                    if (it == col_of.end()) {
                        col = (int32_t)prov.size();
                        col_of.emplace(key, col);
                        prov.push_back(key);
                        seen.push_back(-1);
                    } else col = it->second;
                    if (j < (int32_t)hint.size()) hint[j] = col; else hint.push_back(col);
                }
                if (seen[col] == rid)
                    return input_error(err, "read at :index %d observes key %d twice", h->index[e], key);
                seen[col] = rid;
            }
            H.r_shard.push_back(s);
            H.r_inv.push_back(inv);
            H.r_comp.push_back(pos);
            H.r_ntrip.push_back(nt);
            H.r_ev.push_back(e);
            H.r_poff.push_back(off);
            H.n_reads[s]++;
            H.min_trip[s] = std::min(H.min_trip[s], nt);
        }
        std::sort(prov.begin(), prov.end());
        H.n_keys[s] = (int32_t)prov.size();
        H.keys.insert(H.keys.end(), prov.begin(), prov.end());
        H.key_off[s + 1] = (int64_t)H.keys.size();
        std::fill(seen.begin(), seen.end(), -1);   // read ids only grow, but keep the table tidy per shard
        seen.resize(0);
    }
    return 0;
}

// values of read r by column (the shard's sorted keys)
inline void mono_row(const jtb_history* h, const MonoHost& H, int32_t r, std::vector<int64_t>& out) {
    const int32_t s = H.r_shard[r], K = H.n_keys[s];
    const int32_t* kt = H.keys.data() + H.key_off[s];
    out.assign(K, 0);
    const int32_t* p = h->payload + H.r_poff[r];
    for (int32_t j = 0; j < H.r_ntrip[r]; ++j) out[mono_col(kt, K, p[3 * j])] = mono_join(p[3 * j + 1], p[3 * j + 2]);
}

// the explanation of the edge x -> y: the smallest key with a strict increase, else real time
inline void mono_explain(const jtb_history* h, const MonoHost& H, int32_t x, int32_t y, int realtime,
                         jtb_mono_shard& o, int slot) {
    std::vector<int64_t> vx, vy;
    mono_row(h, H, x, vx);
    mono_row(h, H, y, vy);
    const int32_t s = H.r_shard[x];
    const int64_t base = h->shard_off[s];
    o.edge_kind[slot] = JTB_MONO_EDGE_NONE;
    o.edge_key[slot] = -1;
    o.edge_value[slot] = o.edge_value2[slot] = 0;
    for (size_t c = 0; c < vx.size(); ++c)
        if (vx[c] < vy[c]) {
            o.edge_kind[slot] = JTB_MONO_EDGE_MONOTONIC;
            o.edge_key[slot] = H.keys[H.key_off[s] + c];
            o.edge_value[slot] = vx[c];
            o.edge_value2[slot] = vy[c];
            return;
        }
    if (realtime && H.r_comp[x] < H.r_inv[y]) {
        o.edge_kind[slot] = JTB_MONO_EDGE_REALTIME;
        o.edge_value[slot] = h->index[base + H.r_comp[x]];
        o.edge_value2[slot] = h->index[base + H.r_inv[y]];
    }
}

inline int run_monotonic_keys(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h, int32_t flags,
                              jtb_mono_shard* shards, jtb_mono_result* out, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    if (int rc = check_history(h, false, err)) return rc;
    const int realtime = !(flags & JTB_MONO_NO_REALTIME);
    const int32_t S = h->n_shards;
    MonoHost H;
    if (int rc = mono_host_pass(h, H, err)) return rc;
    memset(out, 0, sizeof *out);
    // shards that go to the device: every read observes every key of the shard, and there are two reads or more
    std::vector<char> dev(S, 0);
    for (int32_t s = 0; s < S; ++s) {
        jtb_mono_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_reads = H.n_reads[s];
        o.n_keys = H.n_keys[s];
        o.witness_index = o.partner_index = -1;
        o.edge_key[0] = o.edge_key[1] = -1;
        if (H.n_reads[s] > 0 && H.min_trip[s] < H.n_keys[s]) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_PARTIAL_READ;
        } else if (H.n_reads[s] >= 2) dev[s] = 1;
        out->n_reads += H.n_reads[s];
    }
    // the device's reads (ids compacted over the shards that go there)
    std::vector<int32_t> d_of;   // device id -> host read id
    std::vector<int32_t> shard_v, inv_v, comp_v, cidx_v;
    std::vector<int64_t> poff_v, row_v;
    int64_t cells = 0;
    for (int32_t r = 0; r < (int32_t)H.r_shard.size(); ++r) {
        const int32_t s = H.r_shard[r];
        if (!dev[s]) continue;
        d_of.push_back(r);
        shard_v.push_back(s);
        inv_v.push_back(H.r_inv[r]);
        comp_v.push_back(H.r_comp[r]);
        cidx_v.push_back(h->index[H.r_ev[r]]);
        poff_v.push_back(H.r_poff[r]);
        row_v.push_back(cells);
        cells += H.n_keys[s];
    }
    const int32_t m = (int32_t)d_of.size();
    float ms_a = 0, ms_b = 0;
    if (m > 0) {
        CallAllocs A;
        MonoDev d;
        d.m = m;
        int64_t* V;
        if (A.alloc(&V, (size_t)cells) != cudaSuccess) {
            err = "cannot allocate the dense value matrix (" + std::to_string((size_t)cells * sizeof(int64_t)) +
                  " bytes on the device)";
            return -3;
        }
        d.V = V;
        const int32_t *payload, *cidx, *keys;
        const int64_t *poff, *key_off;
        MonoKey *key0, *key1;
        MonoSuffix *rev, *scan;
        int32_t *id0, *id1, *bound, *bad, *lo, *hi, *wit;
        unsigned long long* pkey;
        uint8_t* tmp;
        JTB_OK(A.put(&payload, h->payload, (size_t)h->n_payload, st));
        JTB_OK(A.put(&poff, poff_v, st)); JTB_OK(A.put(&d.row, row_v, st));
        JTB_OK(A.put(&d.shard, shard_v, st)); JTB_OK(A.put(&d.inv, inv_v, st)); JTB_OK(A.put(&d.comp, comp_v, st));
        JTB_OK(A.put(&cidx, cidx_v, st));
        JTB_OK(A.put(&d.n_keys, H.n_keys, st)); JTB_OK(A.put(&key_off, H.key_off, st));
        JTB_OK(A.put(&keys, H.keys, st));
        JTB_OK(A.alloc(&key0, m)); JTB_OK(A.alloc(&key1, m));
        JTB_OK(A.alloc(&id0, m)); JTB_OK(A.alloc(&id1, m));
        JTB_OK(A.alloc(&rev, m)); JTB_OK(A.alloc(&scan, m));
        JTB_OK(A.alloc(&bound, S)); JTB_OK(A.alloc(&bad, S));
        JTB_OK(A.alloc(&lo, S)); JTB_OK(A.alloc(&hi, S)); JTB_OK(A.alloc(&wit, S));
        JTB_OK(A.alloc(&pkey, S));
        d.ord = id1;
        size_t tmp_sort = 0, tmp_scan = 0;
        JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, key0, key1, id0, id1, m, MonoKeyDecomposer{}, st));
        JTB_OK(cub::DeviceScan::InclusiveScan(nullptr, tmp_scan, rev, scan, MonoSuffixMin{}, m, st));
        const size_t tmp_bytes = std::max(tmp_sort, tmp_scan);
        JTB_OK(A.alloc(&tmp, tmp_bytes));

        const unsigned warp_grid = (unsigned)(((int64_t)m * 32 + 255) / 256);
        const unsigned thr_grid = (unsigned)(((int64_t)m + 255) / 256);
        const unsigned sh_grid = (unsigned)((S + 255) / 256);
        auto decide = [&]() -> int {
            mono_suffix_init<<<thr_grid, 256, 0, st>>>(d, bound, rev);
            size_t tb = tmp_bytes;
            JTB_OK(cub::DeviceScan::InclusiveScan(tmp, tb, rev, scan, MonoSuffixMin{}, m, st));
            mono_check<<<warp_grid, 256, 0, st>>>(d, bound, scan, realtime, bad);
            return 0;
        };

        JTB_OK(cudaEventRecord(ev0, st));
        mono_scatter<<<warp_grid, 256, 0, st>>>(m, payload, poff, d.shard, d.inv, d.row, d.n_keys, key_off, keys, V,
                                                key0, id0);
        size_t tb = tmp_bytes;
        JTB_OK(cub::DeviceRadixSort::SortPairs(tmp, tb, key0, key1, id0, id1, m, MonoKeyDecomposer{}, st));
        mono_bound_all<<<sh_grid, 256, 0, st>>>(S, bound, bad);
        if (decide()) return -1;
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<int32_t> bad_h(S, 0);
        JTB_OK(cudaMemcpyAsync(bad_h.data(), bad, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms_a, ev0, ev1));

        // witness and partner of the INVALID shards
        std::vector<int32_t> lo_h(S, 0), hi_h(S, 0);
        int64_t widest = 0;
        bool any = false;
        for (int32_t s = 0; s < S; ++s)
            if (dev[s] && bad_h[s]) {
                shards[s].valid = JTB_INVALID;
                hi_h[s] = (int32_t)(h->shard_off[s + 1] - h->shard_off[s] - 1);
                widest = std::max<int64_t>(widest, hi_h[s] + 1);
                any = true;
            }
        if (any) {
            int rounds = 0;
            while ((1ll << rounds) < widest) ++rounds;
            JTB_OK(cudaEventRecord(ev0, st));
            JTB_OK(cudaMemcpyAsync(lo, lo_h.data(), (size_t)S * 4, cudaMemcpyHostToDevice, st));
            JTB_OK(cudaMemcpyAsync(hi, hi_h.data(), (size_t)S * 4, cudaMemcpyHostToDevice, st));
            for (int k = 0; k < rounds; ++k) {
                mono_bound_mid<<<sh_grid, 256, 0, st>>>(S, lo, hi, bound, bad);
                if (decide()) return -1;
                mono_bound_update<<<sh_grid, 256, 0, st>>>(S, lo, hi, bound, bad);
            }
            // wpos: the converged bound of an INVALID shard, -1 elsewhere
            std::vector<int32_t> wpos(S, -1);
            JTB_OK(cudaMemcpyAsync(lo_h.data(), lo, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            for (int32_t s = 0; s < S; ++s)
                if (shards[s].valid == JTB_INVALID && dev[s]) wpos[s] = lo_h[s];
            JTB_OK(cudaMemcpyAsync(lo, wpos.data(), (size_t)S * 4, cudaMemcpyHostToDevice, st));
            JTB_OK(cudaMemsetAsync(pkey, 0xff, (size_t)S * 8, st));
            mono_find_witness<<<thr_grid, 256, 0, st>>>(d, lo, wit);
            mono_partner<<<thr_grid, 256, 0, st>>>(d, lo, wit, cidx, realtime, pkey);
            JTB_OK(cudaGetLastError());
            JTB_OK(cudaEventRecord(ev1, st));
            std::vector<int32_t> wit_h(S, -1);
            std::vector<unsigned long long> pkey_h(S, ~0ull);
            JTB_OK(cudaMemcpyAsync(wit_h.data(), wit, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaMemcpyAsync(pkey_h.data(), pkey, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            JTB_OK(cudaEventElapsedTime(&ms_b, ev0, ev1));
            for (int32_t s = 0; s < S; ++s) {
                if (wpos[s] < 0) continue;
                jtb_mono_shard& o = shards[s];
                o.witness_index = h->index[h->shard_off[s] + wpos[s]];
                if (pkey_h[s] == ~0ull) { err = "internal: an INVALID shard has no 2-cycle partner"; return -1; }
                const int32_t w = d_of[wit_h[s]], p = d_of[(int32_t)(pkey_h[s] & 0xffffffffu)];
                o.partner_index = h->index[H.r_ev[p]];
                mono_explain(h, H, p, w, realtime, o, 0);
                mono_explain(h, H, w, p, realtime, o, 1);
            }
        }
    }
    roll_up(out, shards, S, ms_a + ms_b, t0);
    return 0;
}

}  // namespace jtb
