// jtb_transfer_lookups.cuh — K9: the transfer-lookup check (looked-up transfer records held to the transfers clients
// issued and to the counters reads show) on the device.
//
// Semantics (include/jtb_check.h, DESIGN.md "K9 transfer-lookup check").  The reads, their invocations and the shards'
// key tables are K7's host pass (mono_host_pass).  A second host pass pairs every transfer micro-op with its fate and
// every :ok lookup with its invocation, validates them and builds the transfer table and the per-lookup record offsets;
// the records themselves stay where they lie in the payload.  On the device:
//   - a cub radix sort of the transfer table by (shard, id);
//   - a thread per record: binary search of its id, codes 1-4, an atomicMin of its lookup into the transfer's slot
//     (lookups ascend with completion inside a shard, so the smallest lookup is the earliest completion);
//   - a radix sort of the records by (lookup, id): repeated ids are DUPLICATEs, first occurrences the distinct records,
//     which count the "have" side of LOST / VANISHED and build S with int64 atomicAdds;
//   - M per transfer and a sort of (shard, kind, M): a thread per lookup counts the "need" side by binary search;
//   - per observed key a prefix max of S over lookups by completion and a suffix min by invocation;
//   - a warp per read, a lane per triple, against those two;
//   - the witness: a thread per INVALID shard, plus a thread per transfer for the smallest missing id of LOST /
//     VANISHED.
#pragma once
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include <cub/cub.cuh>
#include <cuda/std/tuple>
#include <cuda_runtime.h>

#include "../../include/jtb_check.h"
#include "jtb_call.cuh"
#include "jtb_monotonic.cuh"

namespace jtb {

constexpr uint64_t TL_SIGN = 0x8000000000000000ull;   // id ^ TL_SIGN: unsigned order is signed id order

struct TlTKey {   // a transfer: (shard, id)
    uint32_t shard;
    uint64_t idu;
};
struct TlTKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, uint64_t&> operator()(TlTKey& k) const { return {k.shard, k.idu}; }
};
struct TlRKey {   // a record: (lookup, id)
    uint32_t lookup;
    uint64_t idu;
};
struct TlRKeyDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint32_t&, uint64_t&> operator()(TlRKey& k) const {
        return {k.lookup, k.idu};
    }
};

struct TlDev {
    const int32_t* payload = nullptr;
    // transfers, in sorted (shard, id) order after the sort: tkey / tperm; per original transfer the rest
    int32_t n_t = 0;
    const TlTKey* tkey = nullptr;
    const int32_t* tperm = nullptr;
    const int32_t* t_shard = nullptr;
    const int32_t* t_rec = nullptr;       // (debit, credit, amount) x n_t
    const int32_t* t_inv = nullptr;       // invocation position
    const int32_t* t_okcomp = nullptr;    // :ok completion position, INT_MAX unless :ok
    const int32_t* t_fate = nullptr;      // JTB_T_*, -1 = never completed
    const int32_t* t_iidx = nullptr;
    const int32_t* t_cidx = nullptr;
    const int32_t* t_off = nullptr;       // [n_shards + 1] the shard's range in the sorted order
    // lookups, shard-major, in completion order inside a shard
    int32_t n_l = 0;
    const int32_t* l_shard = nullptr;
    const int32_t* l_inv = nullptr;       // -1 = none
    const int32_t* l_comp = nullptr;
    const int32_t* l_cidx = nullptr;
    const int64_t* l_poff = nullptr;      // payload offset of the records
    const int64_t* rec_base = nullptr;    // [n_l + 1] global record numbers
    const int32_t* lk_off = nullptr;      // [n_shards + 1]
    const int32_t* ib = nullptr;          // lookups with an invocation, sorted by (shard, invocation)
    const int32_t* ib_inv = nullptr;      // their invocation positions
    const int32_t* ib_off = nullptr;      // [n_shards + 1]
    const int64_t* s_base = nullptr;      // [n_shards] first row of S / P (lookups x keys)
    const int64_t* i_base = nullptr;      // [n_shards] first row of N (ib x keys)
    // keys (K7's tables)
    const int32_t* n_keys = nullptr;
    const int64_t* key_off = nullptr;
    const int32_t* keys = nullptr;
    // reads (K7's)
    int32_t m = 0;
    const int64_t* poff = nullptr;
    const int32_t* ntrip = nullptr;
    const int32_t* r_shard = nullptr;
    const int32_t* r_inv = nullptr;
    const int32_t* r_comp = nullptr;
    const int32_t* r_cidx = nullptr;
    // work
    int64_t n_rec = 0;
    int32_t* rec_slot = nullptr;          // [n_rec] sorted transfer slot of the record, -1 = phantom
    const TlRKey* rkey = nullptr;         // [n_rec] sorted by (lookup, id)
    const int32_t* rval = nullptr;        // [n_rec] the record number in that order
    int32_t* mlk = nullptr;               // [n_t] per slot: the earliest lookup returning it, >= n_l none
    int32_t* mv = nullptr;                // [n_t] per slot: M, INT_MAX none
    int32_t* mfrom = nullptr;             // [n_t] per slot: -1 the :ok completion, else the lookup
    const uint64_t* msort = nullptr;      // [n_t] sorted (shard << 33 | kind << 32 | M)
    unsigned long long* have = nullptr;   // [n_l * 2]
    unsigned long long* wid = nullptr;    // [n_l * 5] smallest id ^ TL_SIGN per code 1-5
    int32_t* lk_code = nullptr;           // [n_l]
    unsigned long long* S = nullptr;      // lookups x keys, int64 sums (two's complement)
    int64_t* P = nullptr;                 // prefix max of S by completion
    int64_t* N = nullptr;                 // suffix min of S by invocation
    unsigned long long* count = nullptr;  // [n_shards * 9]
    unsigned long long* wop = nullptr;    // [n_shards] (completion << 32 | op), op = lookup or 0x80000000 | read
};

// sorted slot of id in shard s, -1 when no transfer invoke carries it
__device__ __forceinline__ int32_t tl_find(const TlDev& d, int32_t s, uint64_t idu) {
    int32_t a = d.t_off[s], b = d.t_off[s + 1];
    while (a < b) {
        const int32_t c = (int32_t)(((int64_t)a + b) >> 1);
        if (d.tkey[c].idu < idu) a = c + 1; else b = c;
    }
    return a < d.t_off[s + 1] && d.tkey[a].idu == idu ? a : -1;
}

// column of key in shard s's key table, -1 when no read observes it
__device__ __forceinline__ int32_t tl_col(const TlDev& d, int32_t s, int64_t key) {
    const int32_t* kt = d.keys + d.key_off[s];
    int32_t a = 0, b = d.n_keys[s];   // mono_col's search for an int64 key: 2 * account + 1 may leave the int32 range
    while (a < b) {
        const int32_t c = (a + b) >> 1;
        if (kt[c] < key) a = c + 1; else b = c;
    }
    return a < d.n_keys[s] && kt[a] == key ? a : -1;
}

__device__ __forceinline__ int32_t tl_lookup_of(const TlDev& d, int64_t g) {   // the lookup holding record g
    int32_t a = 0, b = d.n_l;   // last l with rec_base[l] <= g
    while (b - a > 1) {
        const int32_t c = (a + b) >> 1;
        if (d.rec_base[c] <= g) a = c; else b = c;
    }
    return a;
}

__device__ __forceinline__ const int32_t* tl_rec(const TlDev& d, int32_t l, int64_t g) {
    return d.payload + d.l_poff[l] + 5 * (g - d.rec_base[l]);
}

__device__ __forceinline__ void tl_flag(const TlDev& d, int32_t s, int32_t l, int code, uint64_t idu) {
    atomicAdd(&d.count[s * JTB_TL_KINDS + code - 1], 1ull);
    atomicMin(&d.wid[(int64_t)l * 5 + code - 1], (unsigned long long)idu);
}

__global__ void tl_tkeys(int32_t n, const int32_t* __restrict__ t_shard, const int64_t* __restrict__ t_id,
                         TlTKey* __restrict__ key, int32_t* __restrict__ ids) {
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    key[t] = TlTKey{(uint32_t)t_shard[t], (uint64_t)t_id[t] ^ TL_SIGN};
    ids[t] = (int32_t)t;
}

// thread per record: codes 1-4, the record's slot, the earliest lookup per slot, the (lookup, id) sort key
__global__ void tl_records(TlDev d, TlRKey* __restrict__ rkey, int32_t* __restrict__ rval) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= d.n_rec) return;
    const int32_t l = tl_lookup_of(d, g), s = d.l_shard[l];
    const int32_t* r = tl_rec(d, l, g);
    const uint64_t idu = (uint64_t)mono_join(r[0], r[1]) ^ TL_SIGN;
    const int32_t slot = tl_find(d, s, idu);
    d.rec_slot[g] = slot;
    rkey[g] = TlRKey{(uint32_t)l, idu};
    rval[g] = (int32_t)g;
    if (slot < 0) { tl_flag(d, s, l, JTB_TL_PHANTOM, idu); return; }
    const int32_t t = d.tperm[slot];
    const int32_t* q = d.t_rec + 3 * (int64_t)t;
    if (q[0] != r[2] || q[1] != r[3] || q[2] != r[4]) tl_flag(d, s, l, JTB_TL_MISMATCH, idu);
    if (d.t_fate[t] == JTB_T_FAIL) tl_flag(d, s, l, JTB_TL_FAILED_VISIBLE, idu);
    if (d.t_inv[t] > d.l_comp[l]) tl_flag(d, s, l, JTB_TL_FUTURE, idu);
    atomicMin(&d.mlk[slot], l);
}

// thread per transfer slot: M, where it came from, and the (shard, kind, M) sort key
__global__ void tl_mval(TlDev d, uint64_t* __restrict__ mkey) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.n_t) return;
    const int32_t t = d.tperm[i], l = d.mlk[i];
    int32_t m = d.t_okcomp[t], from = -1;
    if (l < d.n_l && d.l_comp[l] < m) { m = d.l_comp[l]; from = l; }
    d.mv[i] = m;
    d.mfrom[i] = from;
    mkey[i] = (uint64_t)(uint32_t)d.t_shard[t] << 33 | (uint64_t)(from >= 0) << 32 | (uint32_t)m;
}

// thread per record in (lookup, id) order: DUPLICATE, the "have" counts and S over the distinct ids
__global__ void tl_distinct(TlDev d) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.n_rec) return;
    const TlRKey k = d.rkey[i];
    const int32_t l = (int32_t)k.lookup, s = d.l_shard[l];
    if (i > 0 && d.rkey[i - 1].lookup == k.lookup && d.rkey[i - 1].idu == k.idu) {
        tl_flag(d, s, l, JTB_TL_DUPLICATE, k.idu);
        return;
    }
    const int32_t g = d.rval[i], slot = d.rec_slot[g];
    if (slot >= 0 && d.mv[slot] < d.l_inv[l]) atomicAdd(&d.have[2 * (int64_t)l + (d.mfrom[slot] >= 0)], 1ull);
    const int32_t* r = tl_rec(d, l, g);
    const int64_t row = d.s_base[s] + (int64_t)(l - d.lk_off[s]) * d.n_keys[s];
    const int32_t cd = tl_col(d, s, 2 * (int64_t)r[2]), cc = tl_col(d, s, 2 * (int64_t)r[3] + 1);
    if (cd >= 0) atomicAdd(&d.S[row + cd], (unsigned long long)(int64_t)r[4]);
    if (cc >= 0) atomicAdd(&d.S[row + cc], (unsigned long long)(int64_t)r[4]);
}

// first j in [a, b) with key[j] >= x
__device__ __forceinline__ int32_t tl_lower(const uint64_t* key, int32_t a, int32_t b, uint64_t x) {
    while (a < b) {
        const int32_t c = (int32_t)(((int64_t)a + b) >> 1);
        if (key[c] < x) a = c + 1; else b = c;
    }
    return a;
}

// thread per lookup: "need" by counting, the LOST / VANISHED counts, the lookup's smallest code
__global__ void tl_need(TlDev d) {
    const int32_t l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= d.n_l) return;
    const int32_t s = d.l_shard[l], inv = d.l_inv[l];
    int code = 0;
    for (int c = 1; c <= 5 && !code; ++c)
        if (d.wid[(int64_t)l * 5 + c - 1] != ~0ull) code = c;
    if (inv >= 0)
        for (int b = 0; b < 2; ++b) {
            const uint64_t base = (uint64_t)(uint32_t)s << 33 | (uint64_t)b << 32;
            const int64_t need = tl_lower(d.msort, d.t_off[s], d.t_off[s + 1], base | (uint32_t)inv) -
                                 tl_lower(d.msort, d.t_off[s], d.t_off[s + 1], base);
            const int64_t miss = need - (int64_t)d.have[2 * (int64_t)l + b];
            if (miss > 0) {
                atomicAdd(&d.count[s * JTB_TL_KINDS + JTB_TL_LOST + b - 1], (unsigned long long)miss);
                if (!code) code = JTB_TL_LOST + b;
            }
        }
    d.lk_code[l] = code;
    if (code) atomicMin(&d.wop[s], (unsigned long long)(uint32_t)d.l_comp[l] << 32 | (uint32_t)l);
}

// thread per (shard, observed key): P = prefix max of S over the shard's lookups by completion, N = suffix min over
// those with an invocation by invocation
__global__ void tl_extremes(TlDev d, int32_t n_slots, const int32_t* __restrict__ slot_shard) {
    const int32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_slots) return;
    const int32_t s = slot_shard[q], K = d.n_keys[s], col = q - (int32_t)d.key_off[s];
    int64_t run = INT64_MIN;
    for (int32_t l = d.lk_off[s]; l < d.lk_off[s + 1]; ++l) {
        const int64_t row = d.s_base[s] + (int64_t)(l - d.lk_off[s]) * K;
        run = max(run, (int64_t)d.S[row + col]);
        d.P[row + col] = run;
    }
    run = INT64_MAX;
    for (int32_t j = d.ib_off[s + 1] - 1; j >= d.ib_off[s]; --j) {
        const int32_t l = d.ib[j];
        run = min(run, (int64_t)d.S[d.s_base[s] + (int64_t)(l - d.lk_off[s]) * K + col]);
        d.N[d.i_base[s] + (int64_t)(j - d.ib_off[s]) * K + col] = run;
    }
}

// the lookups a read is held to: nb = those completed before its invocation (a prefix in completion order), ja = the
// first, in invocation order, invoked after its completion
__device__ __forceinline__ void tl_span(const TlDev& d, int32_t r, int32_t s, int32_t& nb, int32_t& ja) {
    const int32_t iv = d.r_inv[r], cp = d.r_comp[r];
    int32_t a = d.lk_off[s], b = d.lk_off[s + 1];
    if (iv < 0) b = a;
    while (a < b) {
        const int32_t c = (a + b) >> 1;
        if (d.l_comp[c] < iv) a = c + 1; else b = c;
    }
    nb = a - d.lk_off[s];
    a = d.ib_off[s];
    b = d.ib_off[s + 1];
    while (a < b) {
        const int32_t c = (a + b) >> 1;
        if (d.ib_inv[c] <= cp) a = c + 1; else b = c;
    }
    ja = a;
}

// warp per read, lane per triple: BELOW against P of the last lookup completed before it, ABOVE against N of the
// first lookup invoked after it
__global__ void tl_reads(TlDev d) {
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= d.m) return;
    const int32_t r = (int32_t)w, s = d.r_shard[r], K = d.n_keys[s], nt = d.ntrip[r];
    int32_t nb, ja;
    tl_span(d, r, s, nb, ja);
    if (nb == 0 && ja == d.ib_off[s + 1]) return;   // no lookup holds it
    const int32_t* p = d.payload + d.poff[r];
    const int64_t prow = d.s_base[s] + (int64_t)(nb - 1) * K, nrow = d.i_base[s] + (int64_t)(ja - d.ib_off[s]) * K;
    unsigned below = 0, above = 0;
    for (int32_t j = lane; j < nt; j += 32) {
        const int32_t col = tl_col(d, s, p[3 * j]);
        const int64_t v = mono_join(p[3 * j + 1], p[3 * j + 2]);
        below += nb > 0 && v < d.P[prow + col];
        above += ja < d.ib_off[s + 1] && v > d.N[nrow + col];
    }
    for (int o = 16; o; o >>= 1) {
        below += __shfl_down_sync(0xffffffffu, below, o);
        above += __shfl_down_sync(0xffffffffu, above, o);
    }
    if (lane == 0 && (below || above)) {
        if (below) atomicAdd(&d.count[s * JTB_TL_KINDS + JTB_TL_READ_BELOW_LOOKUP - 1], (unsigned long long)below);
        if (above) atomicAdd(&d.count[s * JTB_TL_KINDS + JTB_TL_READ_ABOVE_LOOKUP - 1], (unsigned long long)above);
        atomicMin(&d.wop[s], (unsigned long long)(uint32_t)d.r_comp[r] << 32 | (0x80000000u | (uint32_t)r));
    }
}

struct TlWitness {
    int32_t kind, key, related, scan;   // scan: the lookup whose smallest missing id tl_missing finds, -1
    int64_t id, value, bound;
    int32_t op_cidx, pad;
};

// thread per shard with a witness op
__global__ void tl_explain(TlDev d, int32_t n_shards, TlWitness* __restrict__ out) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_shards || d.wop[s] == ~0ull) return;
    const uint32_t op = (uint32_t)(d.wop[s] & 0xffffffffu);
    TlWitness o{0, -1, -1, -1, 0, 0, 0, 0, 0};
    if (!(op & 0x80000000u)) {
        const int32_t l = (int32_t)op, code = d.lk_code[l];
        o.kind = code;
        o.op_cidx = d.l_cidx[l];
        if (code <= JTB_TL_DUPLICATE) {
            const uint64_t idu = d.wid[(int64_t)l * 5 + code - 1];
            o.id = (int64_t)(idu ^ TL_SIGN);
            if (code != JTB_TL_PHANTOM && code != JTB_TL_DUPLICATE) o.related = d.t_iidx[d.tperm[tl_find(d, s, idu)]];
        } else {
            o.scan = l;
        }
        out[s] = o;
        return;
    }
    const int32_t r = (int32_t)(op & 0x7fffffffu), K = d.n_keys[s];
    int32_t nb, ja;
    tl_span(d, r, s, nb, ja);
    const int32_t* p = d.payload + d.poff[r];
    const int64_t prow = d.s_base[s] + (int64_t)(nb - 1) * K, nrow = d.i_base[s] + (int64_t)(ja - d.ib_off[s]) * K;
    int32_t bcol = INT_MAX, acol = INT_MAX;
    for (int32_t j = 0; j < d.ntrip[r]; ++j) {
        const int32_t col = tl_col(d, s, p[3 * j]);
        const int64_t v = mono_join(p[3 * j + 1], p[3 * j + 2]);
        if (nb > 0 && v < d.P[prow + col]) bcol = min(bcol, col);
        if (ja < d.ib_off[s + 1] && v > d.N[nrow + col]) acol = min(acol, col);
    }
    const bool below = bcol != INT_MAX;
    const int32_t col = below ? bcol : acol, key = d.keys[d.key_off[s] + col];
    int64_t v = 0;
    for (int32_t j = 0; j < d.ntrip[r]; ++j)
        if (p[3 * j] == key) v = mono_join(p[3 * j + 1], p[3 * j + 2]);
    o.kind = below ? JTB_TL_READ_BELOW_LOOKUP : JTB_TL_READ_ABOVE_LOOKUP;
    o.key = key;
    o.value = v;
    o.op_cidx = d.r_cidx[r];
    const int64_t base = d.s_base[s];
    if (below) {
        o.bound = d.P[prow + col];
        for (int32_t l = d.lk_off[s]; l < d.lk_off[s] + nb; ++l)
            if ((int64_t)d.S[base + (int64_t)(l - d.lk_off[s]) * K + col] > v) { o.related = d.l_cidx[l]; break; }
    } else {
        o.bound = d.N[nrow + col];
        for (int32_t j = ja; j < d.ib_off[s + 1]; ++j) {
            const int32_t l = d.ib[j];
            if ((int64_t)d.S[base + (int64_t)(l - d.lk_off[s]) * K + col] < v) { o.related = d.l_cidx[l]; break; }
        }
    }
    out[s] = o;
}

// thread per transfer slot of a shard whose witness is LOST / VANISHED: is it one the witness lookup misses?
__global__ void tl_missing(TlDev d, const TlWitness* __restrict__ wit, unsigned long long* __restrict__ mid) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= d.n_t) return;
    const int32_t s = d.t_shard[d.tperm[i]];
    if (d.wop[s] == ~0ull) return;
    const int32_t l = wit[s].scan;
    if (l < 0 || !(d.mv[i] < d.l_inv[l]) || JTB_TL_LOST + (d.mfrom[i] >= 0) != wit[s].kind) return;
    const uint64_t idu = d.tkey[i].idu;
    int64_t a = d.rec_base[l], b = d.rec_base[l + 1];
    while (a < b) {
        const int64_t c = (a + b) >> 1;
        if (d.rkey[c].idu < idu) a = c + 1; else b = c;
    }
    if (a < d.rec_base[l + 1] && d.rkey[a].idu == idu) return;
    atomicMin(&mid[s], (unsigned long long)idu);
}

__global__ void tl_missing_related(TlDev d, int32_t n_shards, const unsigned long long* __restrict__ mid,
                                   TlWitness* __restrict__ wit) {
    const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_shards || d.wop[s] == ~0ull || wit[s].scan < 0) return;
    const int32_t slot = tl_find(d, s, mid[s]);
    wit[s].id = (int64_t)(mid[s] ^ TL_SIGN);
    wit[s].related = d.mfrom[slot] >= 0 ? d.l_cidx[d.mfrom[slot]] : d.t_cidx[d.tperm[slot]];
}

// ---- host ---------------------------------------------------------------------------------------------------------

struct TlHost {
    // transfers, shard-major
    std::vector<int32_t> t_shard, t_rec, t_inv, t_okcomp, t_fate, t_iidx, t_cidx, t_off;
    std::vector<int64_t> t_id;
    // :ok lookups, shard-major, completion order
    std::vector<int32_t> l_shard, l_inv, l_comp, l_cidx, lk_off;
    std::vector<int64_t> l_poff, rec_base;
    std::vector<int32_t> ib, ib_inv, ib_off;
};

// Pair every transfer micro-op with the next event of its process and every :ok lookup with the latest invoke of its
// process, validate them, and lay out the transfer table and the lookups' record offsets.
inline int tl_host_pass(const jtb_history* h, TlHost& T, std::string& err) {
    const int32_t S = h->n_shards;
    T.t_off.assign((size_t)S + 1, 0);
    T.lk_off.assign((size_t)S + 1, 0);
    T.ib_off.assign((size_t)S + 1, 0);
    T.rec_base.push_back(0);
    std::unordered_map<int32_t, int32_t> last_inv;                        // process -> latest invoke position
    std::unordered_map<int32_t, std::pair<size_t, size_t>> open;          // process -> its transfers [a, b)
    std::unordered_set<int64_t> ids;
    for (int32_t s = 0; s < S; ++s) {
        const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
        last_inv.clear();
        open.clear();
        ids.clear();
        for (int64_t e = lo; e < hi; ++e) {
            const int32_t p = h->process[e], pos = (int32_t)(e - lo);
            if (p < 0) continue;
            auto ot = open.find(p);
            if (ot != open.end()) {
                if (h->type[e] != JTB_T_INVOKE)
                    for (size_t t = ot->second.first; t < ot->second.second; ++t) {
                        T.t_fate[t] = h->type[e];
                        T.t_cidx[t] = h->index[e];
                        if (h->type[e] == JTB_T_OK) T.t_okcomp[t] = pos;
                    }
                open.erase(ot);
            }
            const int32_t len = h->payload_len[e];
            const int64_t off = h->payload_off[e];
            if (h->type[e] == JTB_T_INVOKE) {
                last_inv[p] = pos;
                if (h->f[e] != JTB_F_TRANSFER) continue;
                if (len <= 0) return input_error(err, "transfer at :index %d: an invoke without ids", h->index[e]);
                if (len % 5 != 0)
                    return input_error(err, "transfer at :index %d: payload length %d is not a multiple of 5",
                                       h->index[e], len);
                if (off < 0 || off + len > h->n_payload)
                    return input_error(err, "transfer at :index %d: payload out of range", h->index[e]);
                const size_t first = T.t_id.size();
                for (int32_t j = 0; j < len; j += 5) {
                    const int32_t* r = h->payload + off + j;
                    if (r[4] < 0)
                        return input_error(err, "transfer at :index %d: negative amount %d", h->index[e], r[4]);
                    if (r[2] < 0 || r[2] >= (1 << 30) || r[3] < 0 || r[3] >= (1 << 30))
                        return input_error(err, "transfer at :index %d: account outside [0, 2^30)", h->index[e]);
                    const int64_t id = mono_join(r[0], r[1]);
                    if (!ids.insert(id).second)
                        return input_error(err, "transfer at :index %d: id %lld is carried by two transfer invokes",
                                           h->index[e], (long long)id);
                    if (T.t_id.size() >= (size_t)INT_MAX) { err = "more than 2^31-1 transfers"; return -2; }
                    T.t_shard.push_back(s);
                    T.t_id.push_back(id);
                    T.t_rec.insert(T.t_rec.end(), {r[2], r[3], r[4]});
                    T.t_inv.push_back(pos);
                    T.t_okcomp.push_back(INT_MAX);
                    T.t_fate.push_back(-1);
                    T.t_iidx.push_back(h->index[e]);
                    T.t_cidx.push_back(-1);
                }
                open[p] = {first, T.t_id.size()};
                continue;
            }
            if (h->type[e] != JTB_T_OK || h->f[e] != JTB_F_LOOKUP || len < 0) continue;
            if (len % 5 != 0)
                return input_error(err, "lookup at :index %d: payload length %d is not a multiple of 5", h->index[e],
                                   len);
            if (off < 0 || off + len > h->n_payload)
                return input_error(err, "lookup at :index %d: payload out of range", h->index[e]);
            if (T.rec_base.back() + len / 5 > INT_MAX) { err = "more than 2^31-1 lookup records"; return -2; }
            auto it = last_inv.find(p);
            T.l_shard.push_back(s);
            T.l_inv.push_back(it == last_inv.end() ? -1 : it->second);
            T.l_comp.push_back(pos);
            T.l_cidx.push_back(h->index[e]);
            T.l_poff.push_back(off);
            T.rec_base.push_back(T.rec_base.back() + len / 5);
        }
        T.t_off[s + 1] = (int32_t)T.t_id.size();
        T.lk_off[s + 1] = (int32_t)T.l_shard.size();
        // the shard's lookups with an invocation, by invocation (stable: ties keep completion order)
        const size_t ib0 = T.ib.size();
        for (int32_t l = T.lk_off[s]; l < T.lk_off[s + 1]; ++l)
            if (T.l_inv[l] >= 0) T.ib.push_back(l);
        std::stable_sort(T.ib.begin() + ib0, T.ib.end(), [&](int32_t a, int32_t b) { return T.l_inv[a] < T.l_inv[b]; });
        for (size_t j = ib0; j < T.ib.size(); ++j) T.ib_inv.push_back(T.l_inv[T.ib[j]]);
        T.ib_off[s + 1] = (int32_t)T.ib.size();
    }
    return 0;
}

inline int run_transfer_lookups(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const jtb_history* h,
                                int32_t flags, jtb_tl_shard* shards, jtb_tl_result* out, std::string& err) {
    const auto t0 = std::chrono::steady_clock::now();
    if (!h || !shards || !out) { err = "null argument"; return -2; }
    if (flags != 0) { err = "flags must be 0 (reserved)"; return -2; }
    if (int rc = check_history(h, false, err)) return rc;
    const int32_t S = h->n_shards;
    MonoHost H;
    if (int rc = mono_host_pass(h, H, err)) return rc;
    TlHost T;
    if (int rc = tl_host_pass(h, T, err)) return rc;
    // the S / P matrices (lookups x the shard's keys) and N (lookups with an invocation x keys)
    std::vector<int64_t> s_base(S), i_base(S);
    int64_t s_rows = 0, i_rows = 0;
    for (int32_t s = 0; s < S; ++s) {
        s_base[s] = s_rows;
        i_base[s] = i_rows;
        s_rows += (int64_t)(T.lk_off[s + 1] - T.lk_off[s]) * H.n_keys[s];
        i_rows += (int64_t)(T.ib_off[s + 1] - T.ib_off[s]) * H.n_keys[s];
    }
    memset(out, 0, sizeof *out);
    for (int32_t s = 0; s < S; ++s) {
        jtb_tl_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.valid = JTB_VALID;
        o.n_lookups = T.lk_off[s + 1] - T.lk_off[s];
        o.n_records = T.rec_base[T.lk_off[s + 1]] - T.rec_base[T.lk_off[s]];
        o.n_transfers = T.t_off[s + 1] - T.t_off[s];
        o.n_reads = H.n_reads[s];
        o.witness_index = o.key = o.related_index = -1;
        out->n_lookups += o.n_lookups;
        out->n_records += o.n_records;
        out->n_transfers += o.n_transfers;
        out->n_reads += o.n_reads;
    }
    const int32_t m = (int32_t)H.r_shard.size(), nT = (int32_t)T.t_id.size(), nL = (int32_t)T.l_shard.size();
    const int64_t nR = T.rec_base.back();
    float ms = 0;
    if (nL > 0) {   // without an :ok lookup nothing can be violated
        CallAllocs A;
        const size_t slots = H.keys.size();
        std::vector<int32_t> slot_shard(slots), r_cidx(m);
        for (int32_t s = 0; s < S; ++s)
            for (int64_t q = H.key_off[s]; q < H.key_off[s + 1]; ++q) slot_shard[q] = s;
        for (int32_t r = 0; r < m; ++r) r_cidx[r] = h->index[H.r_ev[r]];
        TlDev d;
        d.n_t = nT;
        d.n_l = nL;
        d.m = m;
        d.n_rec = nR;
        const int32_t* sshard;
        const int64_t* tid;
        TlTKey *tk0, *tk;
        TlRKey *rk0, *rk;
        int32_t *tid0, *tperm, *rv0, *rv;
        uint64_t *mk0, *mk;
        TlWitness* wit;
        unsigned long long* mid;
        uint8_t* tmp;
        JTB_OK(A.put(&d.payload, h->payload, (size_t)h->n_payload, st));
        JTB_OK(A.put(&d.poff, H.r_poff, st)); JTB_OK(A.put(&d.ntrip, H.r_ntrip, st)); JTB_OK(A.put(&d.r_shard, H.r_shard, st));
        JTB_OK(A.put(&d.r_inv, H.r_inv, st)); JTB_OK(A.put(&d.r_comp, H.r_comp, st)); JTB_OK(A.put(&d.r_cidx, r_cidx, st));
        JTB_OK(A.put(&d.n_keys, H.n_keys, st)); JTB_OK(A.put(&d.key_off, H.key_off, st)); JTB_OK(A.put(&d.keys, H.keys, st));
        JTB_OK(A.put(&sshard, slot_shard, st));
        JTB_OK(A.put(&d.t_shard, T.t_shard, st)); JTB_OK(A.put(&tid, T.t_id, st)); JTB_OK(A.put(&d.t_rec, T.t_rec, st));
        JTB_OK(A.put(&d.t_inv, T.t_inv, st)); JTB_OK(A.put(&d.t_okcomp, T.t_okcomp, st));
        JTB_OK(A.put(&d.t_fate, T.t_fate, st)); JTB_OK(A.put(&d.t_iidx, T.t_iidx, st));
        JTB_OK(A.put(&d.t_cidx, T.t_cidx, st)); JTB_OK(A.put(&d.t_off, T.t_off, st));
        JTB_OK(A.alloc(&tk0, nT)); JTB_OK(A.alloc(&tk, nT));
        JTB_OK(A.alloc(&tid0, nT)); JTB_OK(A.alloc(&tperm, nT));
        JTB_OK(A.put(&d.l_shard, T.l_shard, st)); JTB_OK(A.put(&d.l_inv, T.l_inv, st)); JTB_OK(A.put(&d.l_comp, T.l_comp, st));
        JTB_OK(A.put(&d.l_cidx, T.l_cidx, st)); JTB_OK(A.put(&d.l_poff, T.l_poff, st));
        JTB_OK(A.put(&d.rec_base, T.rec_base, st)); JTB_OK(A.put(&d.lk_off, T.lk_off, st));
        JTB_OK(A.put(&d.ib, T.ib, st)); JTB_OK(A.put(&d.ib_inv, T.ib_inv, st));
        JTB_OK(A.put(&d.ib_off, T.ib_off, st)); JTB_OK(A.put(&d.s_base, s_base, st));
        JTB_OK(A.put(&d.i_base, i_base, st));
        JTB_OK(A.alloc(&d.rec_slot, nR));
        JTB_OK(A.alloc(&rk0, nR)); JTB_OK(A.alloc(&rk, nR));
        JTB_OK(A.alloc(&rv0, nR)); JTB_OK(A.alloc(&rv, nR));
        JTB_OK(A.alloc(&d.mlk, nT)); JTB_OK(A.alloc(&d.mv, nT)); JTB_OK(A.alloc(&d.mfrom, nT));
        JTB_OK(A.alloc(&mk0, nT)); JTB_OK(A.alloc(&mk, nT));
        JTB_OK(A.alloc(&d.have, (size_t)nL * 2)); JTB_OK(A.alloc(&d.wid, (size_t)nL * 5)); JTB_OK(A.alloc(&d.lk_code, nL));
        if (A.alloc(&d.S, (size_t)s_rows) != cudaSuccess || A.alloc(&d.P, (size_t)s_rows) != cudaSuccess ||
            A.alloc(&d.N, (size_t)i_rows) != cudaSuccess)
            return input_error(err, "the S matrix (%lld lookup x observed-key sums) does not fit on the device",
                               (long long)s_rows);
        JTB_OK(A.alloc(&d.count, (size_t)S * JTB_TL_KINDS)); JTB_OK(A.alloc(&d.wop, S));
        JTB_OK(A.alloc(&wit, S)); JTB_OK(A.alloc(&mid, S));
        d.tkey = tk; d.tperm = tperm;
        d.rkey = rk; d.rval = rv;
        d.msort = mk;
        size_t tmp_t = 0, tmp_r = 0, tmp_m = 0;
        if (nT > 0) {
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_t, tk0, tk, tid0, tperm, nT, TlTKeyDecomposer{}, st));
            JTB_OK(cub::DeviceRadixSort::SortKeys(nullptr, tmp_m, mk0, mk, nT, 0, 64, st));
        }
        if (nR > 0)
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_r, rk0, rk, rv0, rv, (int)nR, TlRKeyDecomposer{}, st));
        const size_t tmp_bytes = std::max({tmp_t, tmp_r, tmp_m});
        JTB_OK(A.alloc(&tmp, tmp_bytes));
        auto grid = [](int64_t n, int per) { return (unsigned)((n + per - 1) / per); };

        JTB_OK(cudaEventRecord(ev0, st));
        JTB_OK(cudaMemsetAsync(d.mlk, 0x7f, (size_t)nT * 4, st));   // 0x7f7f7f7f > any lookup id: "none"
        JTB_OK(cudaMemsetAsync(d.have, 0, (size_t)nL * 16, st));
        JTB_OK(cudaMemsetAsync(d.wid, 0xff, (size_t)nL * 40, st));
        JTB_OK(cudaMemsetAsync(d.S, 0, (size_t)s_rows * 8, st));
        JTB_OK(cudaMemsetAsync(d.count, 0, (size_t)S * JTB_TL_KINDS * 8, st));
        JTB_OK(cudaMemsetAsync(d.wop, 0xff, (size_t)S * 8, st));
        JTB_OK(cudaMemsetAsync(mid, 0xff, (size_t)S * 8, st));
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
            tl_mval<<<grid(nT, 256), 256, 0, st>>>(d, mk0);
            tb = tmp_bytes;
            JTB_OK(cub::DeviceRadixSort::SortKeys(tmp, tb, mk0, mk, nT, 0, 64, st));
        }
        if (nR > 0) tl_distinct<<<grid(nR, 256), 256, 0, st>>>(d);
        tl_need<<<grid(nL, 128), 128, 0, st>>>(d);
        if (slots > 0) tl_extremes<<<grid((int64_t)slots, 128), 128, 0, st>>>(d, (int32_t)slots, sshard);
        if (m > 0) tl_reads<<<grid((int64_t)m * 32, 256), 256, 0, st>>>(d);
        tl_explain<<<grid(S, 128), 128, 0, st>>>(d, S, wit);
        if (nT > 0) tl_missing<<<grid(nT, 256), 256, 0, st>>>(d, wit, mid);
        tl_missing_related<<<grid(S, 128), 128, 0, st>>>(d, S, mid, wit);
        JTB_OK(cudaGetLastError());
        JTB_OK(cudaEventRecord(ev1, st));
        std::vector<unsigned long long> count((size_t)S * JTB_TL_KINDS), wop(S);
        std::vector<TlWitness> wit_h(S);
        JTB_OK(cudaMemcpyAsync(count.data(), d.count, count.size() * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(wop.data(), d.wop, (size_t)S * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(wit_h.data(), wit, (size_t)S * sizeof(TlWitness), cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));
        for (int32_t s = 0; s < S; ++s) {
            jtb_tl_shard& o = shards[s];
            for (int k = 0; k < JTB_TL_KINDS; ++k) {
                o.count_by_kind[k] = (int64_t)count[(size_t)s * JTB_TL_KINDS + k];
                out->n_violations += o.count_by_kind[k];
            }
            if (wop[s] == ~0ull) continue;
            const TlWitness& w = wit_h[s];
            o.valid = JTB_INVALID;
            o.witness_index = w.op_cidx;
            o.kind = w.kind;
            o.transfer_id = w.id;
            o.key = w.key;
            o.related_index = w.related;
            o.value = w.value;
            o.bound = w.bound;
        }
    }
    roll_up(out, shards, S, ms, t0);
    return 0;
}

}  // namespace jtb
