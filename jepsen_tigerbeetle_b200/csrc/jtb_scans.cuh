// jtb_scans.cuh — the single-pass checkers on the hot path as HBM-streaming kernels.
//
//  K4 set_full:    jepsen.checker/set-full as called at src/tigerbeetle/workloads/set_full.clj:157
//                  ({:linearizable? true}); semantics SURVEY.md A.3.  Column-scan formulation: for
//                  element e (tracked from its last :add :invoke at index i_e) over :ok reads r with
//                  ok_idx[r] > i_e:
//                      last_present = max inv_idx[r] with e in r ; last_absent = max inv_idx[r] with e not in r
//                      known = min(first :add :ok after i_e, min ok_idx[r] with e in r)
//                  Stage A builds the read-major bit-matrix P[r][e] from the CSR id lists (binary search of each
//                  id in the shard's sorted element table, atomicOr); stage B scans columns (one thread per
//                  element, 32 elements share each 4 B word => coalesced broadcast loads); stage C classifies.
//  K5 bank_totals: src/tigerbeetle/tests/ledger.clj:127-192 (check-op precedence unexpected-key > nil-balance >
//                  wrong-total > negative-value; aggregation; err-badness :116-125).
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/jtb_check.h"
#include "jtb_call.cuh"

namespace jtb {

// =================================================================================================
// set-full
// =================================================================================================
struct SfRead {        // one :ok read (device), in completion (:ok index) order within its shard
    int32_t inv_idx, ok_idx;
    int64_t inv_time, ok_time;
    int64_t pl_off;    // into payload
    int32_t pl_len;
    int32_t shard;     // bit 31 set: :final? read
    int32_t n_elig;    // elements of the shard tracked before this read completed: positions [0, n_elig)
    int32_t pad;
};
constexpr int32_t SF_FINAL_BIT = (int32_t)0x80000000;
struct SfShard {       // device
    int64_t elem_off;  // into element arrays
    int32_t n_elems;
    int32_t n_reads;
    int64_t read_off;  // into reads
    int64_t bits_off;  // into bit matrix (uint32 words); row stride = words_per_row
    int32_t words_per_row;
    int32_t id_min;    // direct id -> position table: lut[id - id_min] (lut_len > 0), else binary search
    int64_t lut_off;
    int32_t lut_len;
    int32_t pad;
    int64_t sorted_off;  // (id, position) pairs sorted by id, for the binary search (lut_len == 0)
};
struct SfElem {        // device, by POSITION = order of the tracking :add :invoke within the shard
    int32_t id;
    int32_t add_inv_idx;   // last :add :invoke of this value
    int32_t add_ok_idx;    // first :add :ok after it, INT32_MAX if none
    int32_t order;         // creation order (output position within the shard)
    int64_t add_ok_time;
};
struct SfAcc {         // per element accumulators (device)
    unsigned long long last_present;  // (inv_idx+1) << 32 | read id   (0 = none)
    unsigned long long last_absent;
    unsigned long long known_read;    // min: ok_idx << 32 | read id    (~0 = none)
    int dup_max;
    int pad;
};

__device__ __forceinline__ int sf_position(const SfShard& sd, const int32_t* __restrict__ lut,
                                           const int2* __restrict__ sorted, int32_t id) {
    if (sd.lut_len > 0) {
        const int64_t k = (int64_t)id - sd.id_min;
        return (k >= 0 && k < sd.lut_len) ? __ldg(lut + sd.lut_off + k) : -1;
    }
    const int2* tb = sorted + sd.sorted_off;
    int lo = 0, hi = sd.n_elems - 1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const int2 v = __ldg(tb + mid);
        if (v.x == id) return v.y;
        if (v.x < id) lo = mid + 1; else hi = mid - 1;
    }
    return -1;
}

__global__ void sf_init_acc(SfAcc* __restrict__ acc, int64_t n) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g < n) acc[g] = SfAcc{0, 0, ~0ull, 0, 0};
}

// Stage A: the read-major bit-matrix P[r][position] from the id lists.  One warp per read.
// read_flag bit 0: some tracked id occurs twice; bit 1: the read holds ids that were never :add-invoked in this key.
__global__ void sf_build_bits(const SfRead* __restrict__ reads, int64_t n_reads, const SfShard* __restrict__ shards,
                              const int32_t* __restrict__ lut, const int2* __restrict__ sorted,
                              const int32_t* __restrict__ payload, uint32_t* __restrict__ bits, int* __restrict__ read_flag) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_reads) return;
    const SfRead rd = reads[r];
    const SfShard sd = shards[rd.shard & ~SF_FINAL_BIT];
    uint32_t* rowbits = bits + sd.bits_off + (r - sd.read_off) * (int64_t)sd.words_per_row;
    int fl = 0;
    for (int i = lane; i < rd.pl_len; i += 32) {
        const int32_t id = __ldg(payload + rd.pl_off + i);
        const int pos = sf_position(sd, lut, sorted, id);
        if (pos >= 0) {
            const uint32_t bit = 1u << (pos & 31);
            const uint32_t old = atomicOr(rowbits + (pos >> 5), bit);
            fl |= (old & bit) ? 1 : 0;
        } else {
            fl |= 2;
        }
    }
    fl = __reduce_or_sync(0xffffffffu, fl);
    if (fl && lane == 0) read_flag[r] = fl;
}

// (read-all-invoked-adds) workloads/set_full.clj:51-75 on the same bit-matrix: a :final? :ok read is suspect
// when any tracked element (= any value ever :add-invoked in the sub-history) is absent from it.
// One warp per read; writes the number of missing elements (0 for non-final reads).
__global__ void sf_final_missing(const SfRead* __restrict__ reads, int64_t n_reads, const SfShard* __restrict__ shards,
                                 const uint32_t* __restrict__ bits, int* __restrict__ missing) {
    const int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_reads) return;
    const SfRead rd = reads[r];
    if (!(rd.shard & SF_FINAL_BIT)) { if (lane == 0) missing[r] = 0; return; }
    const SfShard sd = shards[rd.shard & ~SF_FINAL_BIT];
    const uint32_t* rowbits = bits + sd.bits_off + (r - sd.read_off) * (int64_t)sd.words_per_row;
    int zeros = 0;
    for (int w = lane; w < sd.words_per_row; w += 32) {
        const int valid_bits = min(32, sd.n_elems - w * 32);
        const uint32_t m = valid_bits == 32 ? 0xffffffffu : ((1u << valid_bits) - 1);
        zeros += __popc(~rowbits[w] & m);
    }
    for (int o = 16; o > 0; o >>= 1) zeros += __shfl_xor_sync(0xffffffffu, zeros, o);
    if (lane == 0) missing[r] = zeros;
}

// exact multiplicities for the (rare) reads that contain a repeated tracked element
__global__ void sf_count_dups(const SfRead* __restrict__ reads, const int* __restrict__ flagged, int n_flagged,
                              const SfShard* __restrict__ shards, const int32_t* __restrict__ lut,
                              const int2* __restrict__ sorted, const int32_t* __restrict__ payload, SfAcc* __restrict__ acc) {
    if ((int)blockIdx.x >= n_flagged) return;
    const int r = flagged[blockIdx.x];
    const SfRead rd = reads[r];
    const SfShard sd = shards[rd.shard & ~SF_FINAL_BIT];
    for (int i = threadIdx.x; i < rd.pl_len; i += blockDim.x) {
        const int32_t id = payload[rd.pl_off + i];
        int cnt = 0;
        for (int j = 0; j < rd.pl_len; ++j) cnt += payload[rd.pl_off + j] == id;
        if (cnt > 1) {
            const int pos = sf_position(sd, lut, sorted, id);
            if (pos >= 0) atomicMax(&acc[sd.elem_off + pos].dup_max, cnt);
        }
    }
}

constexpr int SF_RCHUNK = 512;   // reads per thread-chunk of the column scan

// Stage B, bit-parallel: one thread owns one 32-element WORD of the matrix for a chunk of reads.  Elements sit in the
// order of their tracking :add :invoke, so "read r may constrain element e" (ok_idx[r] > add_inv[e]) is a PREFIX of
// the positions: n_elig[r].  Pass 1 walks the chunk's reads in DESCENDING invocation order (order_desc): the first
// eligible read that shows a bit set / clear is that element's last_present / last_absent inside the chunk (chunks
// merge by atomicMax); pass 2 walks them in completion order: the first eligible present read is known_read (atomicMin).
// A word stops as soon as all of its 32 elements are settled.
// grid: (word tiles of 128, read chunks chunk0.., shards shard0..); grid.y and grid.z are capped at 65,535, so the host
// launches one slice of at most that many chunks and shards at a time.
constexpr int64_t SF_GRID_YZ_MAX = 65535;
__global__ void __launch_bounds__(128) sf_column_scan(const SfRead* __restrict__ reads, const SfShard* __restrict__ shards,
                                                      const int32_t* __restrict__ order_desc,
                                                      const uint32_t* __restrict__ bits, SfAcc* __restrict__ acc,
                                                      int64_t chunk0, int64_t shard0) {
    const SfShard sd = shards[shard0 + blockIdx.z];
    const int w = blockIdx.x * 128 + threadIdx.x;
    const int64_t r0_64 = (chunk0 + blockIdx.y) * SF_RCHUNK;
    if (blockIdx.x * 128 >= sd.words_per_row || r0_64 >= sd.n_reads) return;
    const int r0 = (int)r0_64;
    const int r1 = min(sd.n_reads, r0 + SF_RCHUNK);
    __shared__ int s_r[SF_RCHUNK], s_inv[SF_RCHUNK], s_elig[SF_RCHUNK];
    const bool live = w < sd.words_per_row;
    const int valid_bits = live ? min(32, sd.n_elems - w * 32) : 0;
    const uint32_t all = valid_bits >= 32 ? 0xffffffffu : ((1u << valid_bits) - 1);
    const uint32_t* col = bits + sd.bits_off + w;
    SfAcc* a = acc + sd.elem_off + (int64_t)w * 32;
    // ---- pass 1: descending invocation order -> last_present / last_absent ------------------------------------
    for (int k = threadIdx.x; k < r1 - r0; k += 128) {
        const int r = order_desc[sd.read_off + r0 + k];
        s_r[k] = r;
        s_inv[k] = reads[sd.read_off + r].inv_idx;
        s_elig[k] = reads[sd.read_off + r].n_elig;
    }
    __syncthreads();
    if (live) {
        uint32_t need_p = all, need_a = all;
        for (int k = 0; k < r1 - r0 && (need_p | need_a); ++k) {
            const int e = s_elig[k] - w * 32;
            if (e <= 0) continue;
            const uint32_t el = e >= 32 ? 0xffffffffu : ((1u << e) - 1);
            const int r = s_r[k];
            const uint32_t wv = __ldg(col + (int64_t)r * sd.words_per_row);
            uint32_t np = wv & el & need_p, na = ~wv & el & need_a;
            need_p &= ~np; need_a &= ~na;
            const unsigned long long iv = ((unsigned long long)(uint32_t)(s_inv[k] + 1) << 32) | (uint32_t)r;
            while (np) { const int b = __ffs(np) - 1; np &= np - 1; atomicMax(&a[b].last_present, iv); }
            while (na) { const int b = __ffs(na) - 1; na &= na - 1; atomicMax(&a[b].last_absent, iv); }
        }
    }
    __syncthreads();
    // ---- pass 2: completion order -> known_read ------------------------------------------------------------------
    for (int k = threadIdx.x; k < r1 - r0; k += 128) {
        s_inv[k] = reads[sd.read_off + r0 + k].ok_idx;
        s_elig[k] = reads[sd.read_off + r0 + k].n_elig;
    }
    __syncthreads();
    if (live) {
        uint32_t need_k = all;
        for (int k = 0; k < r1 - r0 && need_k; ++k) {
            const int e = s_elig[k] - w * 32;
            if (e <= 0) continue;
            const uint32_t el = e >= 32 ? 0xffffffffu : ((1u << e) - 1);
            const int r = r0 + k;
            const uint32_t wv = __ldg(col + (int64_t)r * sd.words_per_row);
            uint32_t nk = wv & el & need_k;
            need_k &= ~nk;
            const unsigned long long kv = ((unsigned long long)(uint32_t)s_inv[k] << 32) | (uint32_t)r;
            while (nk) { const int b = __ffs(nk) - 1; nk &= nk - 1; atomicMin(&a[b].known_read, kv); }
        }
    }
}

struct SfShardOut {   // device per-shard tallies
    int attempt, stable, lost, never_read, stale, duplicated;
    long long stable_lat_max, lost_lat_max;
};

__global__ void sf_classify(const SfRead* __restrict__ reads, const SfShard* __restrict__ shards,
                            const SfElem* __restrict__ elems, const SfAcc* __restrict__ acc, int64_t n_elems_total,
                            const int32_t* __restrict__ elem_shard, uint8_t* __restrict__ outcome,
                            long long* __restrict__ latency_ms, int* __restrict__ dup_count, int32_t* __restrict__ out_id,
                            SfShardOut* __restrict__ tallies) {
    const int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (g >= n_elems_total) return;
    const int s = elem_shard[g];
    const SfShard sd = shards[s];
    const SfElem el = elems[g];
    const SfAcc a = acc[g];
    const bool has_lp = a.last_present != 0, has_la = a.last_absent != 0;
    const int lp_idx = has_lp ? (int)(a.last_present >> 32) - 1 : -1;
    const int la_idx = has_la ? (int)(a.last_absent >> 32) - 1 : -1;
    // known = earliest of (first add :ok after the tracking invoke, first observing read :ok)
    int known_idx = 0x7fffffff;
    long long known_time = 0;
    if (el.add_ok_idx != 0x7fffffff) { known_idx = el.add_ok_idx; known_time = el.add_ok_time; }
    if (a.known_read != ~0ull) {
        const int k = (int)(a.known_read >> 32);
        if (k < known_idx) { known_idx = k; known_time = reads[sd.read_off + (uint32_t)a.known_read].ok_time; }
    }
    const bool has_known = known_idx != 0x7fffffff;
    const bool stable = has_lp && la_idx < lp_idx;
    const bool lost = has_known && has_la && lp_idx < la_idx && known_idx < la_idx;
    int oc = JTB_SF_NEVER_READ;
    long long lat = 0;
    if (stable) {
        const long long stable_time = has_la ? reads[sd.read_off + (uint32_t)a.last_absent].inv_time + 1 : 0;
        const long long d = max(0ll, stable_time - known_time);
        lat = (long long)((double)d / 1e6);  // (long (util/nanos->ms d))
        oc = JTB_SF_STABLE;
        atomicAdd(&tallies[s].stable, 1);
        if (lat > 0) atomicAdd(&tallies[s].stale, 1);
        atomicMax(&tallies[s].stable_lat_max, lat);
    } else if (lost) {
        const long long lost_time = has_lp ? reads[sd.read_off + (uint32_t)a.last_present].inv_time + 1 : 0;
        const long long d = max(0ll, lost_time - known_time);
        lat = (long long)((double)d / 1e6);
        oc = JTB_SF_LOST;
        atomicAdd(&tallies[s].lost, 1);
        atomicMax(&tallies[s].lost_lat_max, lat);
    } else {
        atomicAdd(&tallies[s].never_read, 1);
    }
    if (a.dup_max > 1) atomicAdd(&tallies[s].duplicated, 1);
    // output in creation order within the shard
    const int64_t o = sd.elem_off + el.order;
    outcome[o] = (uint8_t)oc;
    latency_ms[o] = lat;
    dup_count[o] = a.dup_max > 1 ? a.dup_max : 0;
    out_id[o] = el.id;
}

// Device buffers of the set-full pass, cached in the context (grown on demand, reused across calls).
struct SfBuffers {
    struct Buf { void* p = nullptr; size_t cap = 0; } b[20];
    void release() { for (auto& x : b) { if (x.p) cudaFree(x.p); x = Buf(); } }
};

inline int run_set_full(cudaStream_t st, cudaEvent_t e0, cudaEvent_t e1, SfBuffers& B, const jtb_history* h,
                        int linearizable, jtb_setfull_out* out, std::string& err, unsigned long long* stats) {
    const double t_start = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
    const int n_shards = h->n_shards;
    // ---- host pass: tracked elements and :ok reads per shard (O(events)) -----------------------
    std::vector<SfShard> shards(n_shards);
    std::vector<SfElem> elems;
    std::vector<int32_t> elem_shard, lut, order_desc;
    std::vector<int2> sorted;
    std::vector<SfRead> reads;
    int64_t bits_words = 0;
    for (int s = 0; s < n_shards; ++s) {
        struct Tr { int32_t add_inv_idx, add_ok_idx, order; int64_t add_ok_time; };
        std::unordered_map<int32_t, Tr> tracked;
        std::unordered_map<int32_t, std::pair<int32_t, int64_t>> open_reads;  // process -> (inv idx, inv time)
        int n_created = 0;
        const int64_t read_off = (int64_t)reads.size();
        for (int64_t e = h->shard_off[s]; e < h->shard_off[s + 1]; ++e) {
            if (h->process[e] < 0) continue;
            const int type = h->type[e], f = h->f[e];
            if (f == JTB_F_ADD) {
                if (type == JTB_T_INVOKE) tracked[h->a[e]] = Tr{h->index[e], 0x7fffffff, n_created++, 0};
                else if (type == JTB_T_OK) {
                    auto it = tracked.find(h->a[e]);
                    if (it != tracked.end() && it->second.add_ok_idx == 0x7fffffff) {
                        it->second.add_ok_idx = h->index[e];
                        it->second.add_ok_time = h->time_ns[e];
                    }
                }
            } else if (f == JTB_F_READ) {
                const int32_t p = h->process[e];
                if (type == JTB_T_INVOKE) open_reads[p] = {h->index[e], h->time_ns[e]};
                else if (type == JTB_T_FAIL) open_reads.erase(p);
                else if (type == JTB_T_OK) {
                    auto it = open_reads.find(p);
                    if (it == open_reads.end()) { err = "malformed history: read :ok without invoke"; return -3; }
                    SfRead r;
                    r.inv_idx = it->second.first; r.inv_time = it->second.second;
                    r.ok_idx = h->index[e]; r.ok_time = h->time_ns[e];
                    r.pl_off = h->payload_off[e];
                    r.pl_len = std::max(0, (int)h->payload_len[e]);
                    r.shard = s | ((h->flags && (h->flags[e] & JTB_FLAG_FINAL)) ? SF_FINAL_BIT : 0);
                    r.n_elig = 0; r.pad = 0;
                    reads.push_back(r);
                }
            }
        }
        // creation order is dense over the surviving elements; positions follow the tracking :add :invoke
        std::vector<std::pair<int32_t, Tr>> v(tracked.begin(), tracked.end());
        std::sort(v.begin(), v.end(), [](auto& x, auto& y) { return x.second.order < y.second.order; });
        for (size_t i = 0; i < v.size(); ++i) v[i].second.order = (int32_t)i;
        std::sort(v.begin(), v.end(), [](auto& x, auto& y) { return x.second.add_inv_idx < y.second.add_inv_idx; });
        SfShard& sd = shards[s];
        std::memset(&sd, 0, sizeof sd);
        sd.elem_off = (int64_t)elems.size();
        sd.n_elems = (int32_t)v.size();
        sd.read_off = read_off;
        sd.n_reads = (int32_t)(reads.size() - read_off);
        sd.words_per_row = (sd.n_elems + 31) / 32;
        sd.bits_off = bits_words;
        bits_words += (int64_t)sd.words_per_row * sd.n_reads;
        // id -> position: a direct table when the ids are dense (account ids are consecutive integers,
        // workloads/set_full.clj:22-32), a sorted (id, position) table otherwise
        int32_t id_min = 0x7fffffff, id_max = (int32_t)0x80000000;
        for (auto& kv : v) { id_min = std::min(id_min, kv.first); id_max = std::max(id_max, kv.first); }
        const int64_t span = v.empty() ? 0 : (int64_t)id_max - id_min + 1;
        sd.id_min = v.empty() ? 0 : id_min;
        sd.lut_off = (int64_t)lut.size();
        sd.sorted_off = (int64_t)sorted.size();
        if (!v.empty() && span <= 4 * (int64_t)v.size() + 1024) {
            sd.lut_len = (int32_t)span;
            lut.resize(lut.size() + (size_t)span, -1);
            for (size_t i = 0; i < v.size(); ++i) lut[(size_t)sd.lut_off + (size_t)(v[i].first - id_min)] = (int32_t)i;
        } else {
            sd.lut_len = 0;
            const size_t o = sorted.size();
            for (size_t i = 0; i < v.size(); ++i) sorted.push_back(int2{v[i].first, (int)i});
            std::sort(sorted.begin() + o, sorted.end(), [](const int2& x, const int2& y) { return x.x < y.x; });
        }
        std::vector<int32_t> inv_sorted(v.size());
        for (size_t i = 0; i < v.size(); ++i) {
            const auto& kv = v[i];
            inv_sorted[i] = kv.second.add_inv_idx;
            elems.push_back(SfElem{kv.first, kv.second.add_inv_idx, kv.second.add_ok_idx, kv.second.order, kv.second.add_ok_time});
            elem_shard.push_back(s);
        }
        // per read: how many elements were tracked before it completed; reads in descending invocation order
        const size_t o_desc = order_desc.size();
        for (int r = 0; r < sd.n_reads; ++r) {
            SfRead& rd = reads[(size_t)read_off + r];
            rd.n_elig = (int32_t)(std::lower_bound(inv_sorted.begin(), inv_sorted.end(), rd.ok_idx) - inv_sorted.begin());
            order_desc.push_back(r);
        }
        std::sort(order_desc.begin() + o_desc, order_desc.end(), [&](int32_t x, int32_t y) {
            return reads[(size_t)read_off + x].inv_idx > reads[(size_t)read_off + y].inv_idx;
        });
    }
    const int64_t n_elems = (int64_t)elems.size(), n_reads = (int64_t)reads.size();
    if (out->elem_capacity > 0 && out->elem_capacity < n_elems) { err = "elem_capacity too small"; return -4; }
    // ---- device buffers (cached in the context) ----------------------------------------------------
    int nb = 0;
    auto dev = [&](size_t bytes) -> void* {
        SfBuffers::Buf& x = B.b[nb++];
        bytes = std::max<size_t>(bytes, 16);
        if (bytes > x.cap) {
            if (x.p) cudaFree(x.p);
            x.p = nullptr; x.cap = 0;
            if (cudaMalloc(&x.p, bytes + bytes / 8) != cudaSuccess) {
                x.p = nullptr;
                (void)cudaGetLastError();   // the refusal would otherwise stay behind as the thread's last error
                return nullptr;
            }
            x.cap = bytes + bytes / 8;
        }
        return x.p;
    };
    SfShard* d_shards = (SfShard*)dev(n_shards * sizeof(SfShard));
    SfElem* d_elems = (SfElem*)dev(n_elems * sizeof(SfElem));
    int32_t* d_elem_shard = (int32_t*)dev(n_elems * 4);
    SfRead* d_reads = (SfRead*)dev(n_reads * sizeof(SfRead));
    int32_t* d_payload = (int32_t*)dev((size_t)h->n_payload * 4);
    uint32_t* d_bits = (uint32_t*)dev((size_t)bits_words * 4);
    int* d_flag = (int*)dev(n_reads * 4);
    SfAcc* d_acc = (SfAcc*)dev(n_elems * sizeof(SfAcc));
    uint8_t* d_outcome = (uint8_t*)dev(n_elems);
    long long* d_lat = (long long*)dev(n_elems * 8);
    int* d_dup = (int*)dev(n_elems * 4);
    int32_t* d_id = (int32_t*)dev(n_elems * 4);
    SfShardOut* d_tally = (SfShardOut*)dev(n_shards * sizeof(SfShardOut));
    int* d_missing = (int*)dev(n_reads * 4);
    int32_t* d_lut = (int32_t*)dev(lut.size() * 4);
    int2* d_sorted = (int2*)dev(sorted.size() * sizeof(int2));
    int32_t* d_order = (int32_t*)dev(order_desc.size() * 4);
    int* d_flagged = (int*)dev(n_reads * 4);
    for (int i = 0; i < nb; ++i)
        if (!B.b[i].p) { err = "set-full: out of device memory"; return -1; }
    unsigned long long h2d = 0;
    auto up = [&](void* d, const void* src, size_t bytes) -> cudaError_t {
        h2d += bytes;
        return bytes ? cudaMemcpyAsync(d, src, bytes, cudaMemcpyHostToDevice, st) : cudaSuccess;
    };
    JTB_OK(cudaMemsetAsync(d_missing, 0, std::max<size_t>(n_reads * 4, 16), st));
    JTB_OK(up(d_shards, shards.data(), n_shards * sizeof(SfShard)));
    JTB_OK(up(d_elems, elems.data(), n_elems * sizeof(SfElem)));
    JTB_OK(up(d_elem_shard, elem_shard.data(), n_elems * 4));
    JTB_OK(up(d_reads, reads.data(), n_reads * sizeof(SfRead)));
    JTB_OK(up(d_lut, lut.data(), lut.size() * 4));
    JTB_OK(up(d_sorted, sorted.data(), sorted.size() * sizeof(int2)));
    JTB_OK(up(d_order, order_desc.data(), order_desc.size() * 4));
    // the id lists: a true DMA when the caller's buffer is page-locked (jtb_host_alloc / cudaHostRegister), staged
    // through the driver's bounce buffer otherwise
    JTB_OK(up(d_payload, h->payload, (size_t)h->n_payload * 4));
    JTB_OK(cudaEventRecord(e0, st));
    JTB_OK(cudaMemsetAsync(d_bits, 0, std::max<size_t>((size_t)bits_words * 4, 16), st));
    JTB_OK(cudaMemsetAsync(d_flag, 0, std::max<size_t>(n_reads * 4, 16), st));
    JTB_OK(cudaMemsetAsync(d_tally, 0, std::max<size_t>(n_shards * sizeof(SfShardOut), 16), st));
    int launches = 0;
    std::vector<int> flag((size_t)n_reads, 0);
    if (n_elems > 0) {
        sf_init_acc<<<(unsigned)((n_elems + 255) / 256), 256, 0, st>>>(d_acc, n_elems);
        JTB_OK(cudaGetLastError());
        ++launches;
    }
    if (n_reads > 0) {
        // stage A runs even when no shard tracks an element: it is what flags the reads holding untracked ids, whose
        // repeats count as :duplicated (sf_position finds nothing in an empty shard, so no bit is set)
        const int64_t threads = n_reads * 32;
        sf_build_bits<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(d_reads, n_reads, d_shards, d_lut, d_sorted, d_payload, d_bits, d_flag);
        JTB_OK(cudaGetLastError());
        ++launches;
        if (n_elems > 0) {
            int max_w = 0, max_r = 0;
            for (auto& sd : shards) { max_w = std::max(max_w, sd.words_per_row); max_r = std::max(max_r, sd.n_reads); }
            const int64_t n_chunks = (max_r + SF_RCHUNK - 1) / SF_RCHUNK;
            for (int64_t s0 = 0; s0 < n_shards; s0 += SF_GRID_YZ_MAX)
                for (int64_t c0 = 0; c0 < n_chunks; c0 += SF_GRID_YZ_MAX) {
                    dim3 grid((max_w + 127) / 128, (unsigned)std::min(SF_GRID_YZ_MAX, n_chunks - c0),
                              (unsigned)std::min(SF_GRID_YZ_MAX, n_shards - s0));
                    sf_column_scan<<<grid, 128, 0, st>>>(d_reads, d_shards, d_order, d_bits, d_acc, c0, s0);
                    JTB_OK(cudaGetLastError());
                    ++launches;
                }
            sf_final_missing<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(d_reads, n_reads, d_shards, d_bits, d_missing);
            JTB_OK(cudaGetLastError());
            ++launches;
        }
        // duplicates (rare): exact multiplicities for flagged reads
        JTB_OK(cudaMemcpyAsync(flag.data(), d_flag, n_reads * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        std::vector<int> flagged;
        for (int64_t r = 0; r < n_reads; ++r) if (flag[r] & 1) flagged.push_back((int)r);
        if (!flagged.empty()) {
            JTB_OK(cudaMemcpyAsync(d_flagged, flagged.data(), flagged.size() * 4, cudaMemcpyHostToDevice, st));
            sf_count_dups<<<(unsigned)flagged.size(), 128, 0, st>>>(d_reads, d_flagged, (int)flagged.size(), d_shards, d_lut, d_sorted, d_payload, d_acc);
            JTB_OK(cudaGetLastError());
            ++launches;
        }
    }
    if (n_elems > 0) {
        sf_classify<<<(unsigned)((n_elems + 255) / 256), 256, 0, st>>>(d_reads, d_shards, d_elems, d_acc, n_elems, d_elem_shard,
                                                                      d_outcome, d_lat, d_dup, d_id, d_tally);
        JTB_OK(cudaGetLastError());
        ++launches;
    }
    JTB_OK(cudaEventRecord(e1, st));
    std::vector<SfShardOut> tally(n_shards);
    JTB_OK(cudaMemcpyAsync(tally.data(), d_tally, n_shards * sizeof(SfShardOut), cudaMemcpyDeviceToHost, st));
    if (out->elem_capacity > 0 && n_elems > 0) {
        JTB_OK(cudaMemcpyAsync(out->elem_outcome, d_outcome, n_elems, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(out->elem_latency_ms, d_lat, n_elems * 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(out->elem_dup_count, d_dup, n_elems * 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(out->elem_id, d_id, n_elems * 4, cudaMemcpyDeviceToHost, st));
    }
    std::vector<int> h_missing((size_t)n_reads, 0);
    if (n_reads > 0) JTB_OK(cudaMemcpyAsync(h_missing.data(), d_missing, n_reads * 4, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaStreamSynchronize(st));
    float ms = 0;
    JTB_OK(cudaEventElapsedTime(&ms, e0, e1));
    // ids that were never :add-invoked in their key but occur twice in one read: jepsen counts (frequencies v) over
    // every value of a read, so they are :duplicated too.  Such reads are flagged by stage A (never in a healthy
    // history); their id lists are counted here.
    std::vector<int> untracked_dups(n_shards, 0);
    {
        std::vector<std::unordered_map<int32_t, int>> seen(n_shards);
        for (int64_t r = 0; r < n_reads; ++r) {
            if (!(flag[r] & 2)) continue;
            const int s = reads[r].shard & ~SF_FINAL_BIT;
            const SfShard& sd = shards[s];
            std::unordered_map<int32_t, int> cnt;
            for (int i = 0; i < reads[r].pl_len; ++i) {
                const int32_t id = h->payload[reads[r].pl_off + i];
                bool is_tracked;
                if (sd.lut_len > 0) {
                    const int64_t k = (int64_t)id - sd.id_min;
                    is_tracked = k >= 0 && k < sd.lut_len && lut[(size_t)sd.lut_off + (size_t)k] >= 0;
                } else {
                    auto b0 = sorted.begin() + sd.sorted_off, b1 = b0 + sd.n_elems;
                    auto it = std::lower_bound(b0, b1, id, [](const int2& x, int32_t v) { return x.x < v; });
                    is_tracked = it != b1 && it->x == id;
                }
                if (!is_tracked) cnt[id]++;
            }
            for (auto& kv : cnt)
                if (kv.second > 1 && seen[s].emplace(kv.first, 1).second) untracked_dups[s]++;
        }
    }
    // read-all-invoked-adds: suspects = final reads with missing elements; ids enumerated from their bit rows
    std::vector<int> suspect_per_shard(n_shards, 0);
    out->n_suspect = 0;
    out->raia_valid = JTB_VALID;
    {
        int64_t cursor = 0;
        if (out->suspect_capacity > 0) out->suspect_missing_off[0] = 0;
        std::vector<uint32_t> rowbits;
        for (int64_t r = 0; r < n_reads; ++r) {
            if (!h_missing[r]) continue;
            const int s = reads[r].shard & ~SF_FINAL_BIT;
            suspect_per_shard[s]++;
            out->raia_valid = JTB_INVALID;
            if (out->suspect_capacity > 0) {
                if (out->n_suspect >= out->suspect_capacity || cursor + h_missing[r] > out->missing_capacity) {
                    err = "suspect/missing capacity too small";
                    return -4;
                }
                const SfShard& sd = shards[s];
                rowbits.resize(sd.words_per_row);
                JTB_OK(cudaMemcpy(rowbits.data(), d_bits + sd.bits_off + (r - sd.read_off) * (int64_t)sd.words_per_row,
                               (size_t)sd.words_per_row * 4, cudaMemcpyDeviceToHost));
                out->suspect_shard[out->n_suspect] = s;
                out->suspect_index[out->n_suspect] = reads[r].ok_idx;
                const int64_t first = cursor;
                for (int e = 0; e < sd.n_elems; ++e)
                    if (!((rowbits[e >> 5] >> (e & 31)) & 1u)) out->missing_ids[cursor++] = elems[sd.elem_off + e].id;
                std::sort(out->missing_ids + first, out->missing_ids + cursor);
                out->suspect_missing_off[out->n_suspect + 1] = cursor;
            }
            out->n_suspect++;
        }
    }
    out->valid = JTB_VALID;
    out->n_failures = 0;
    if (out->elem_capacity > 0) out->elem_off[0] = 0;
    for (int s = 0; s < n_shards; ++s) {
        jtb_setfull_shard& r = out->shards[s];
        std::memset(&r, 0, sizeof r);
        r.suspect_final_reads = suspect_per_shard[s];
        r.attempt_count = shards[s].n_elems;
        r.stable_count = tally[s].stable; r.lost_count = tally[s].lost; r.never_read_count = tally[s].never_read;
        r.stale_count = tally[s].stale; r.duplicated_count = tally[s].duplicated + untracked_dups[s];
        r.stable_latency_max_ms = tally[s].stable_lat_max; r.lost_latency_max_ms = tally[s].lost_lat_max;
        int valid;
        if (r.lost_count > 0) valid = JTB_INVALID;
        else if (r.stable_count == 0) valid = JTB_UNKNOWN;
        else if (linearizable && r.stale_count > 0) valid = JTB_INVALID;
        else valid = JTB_VALID;
        if (r.duplicated_count > 0) valid = JTB_INVALID;
        r.valid = valid;
        out->valid = std::max(out->valid, valid);
        out->n_failures += valid != JTB_VALID;
        if (out->elem_capacity > 0) out->elem_off[s + 1] = shards[s].elem_off + shards[s].n_elems;
    }
    out->seconds_kernel = ms * 1e-3;
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count() - t_start;
    if (stats) {
        stats[11] = (unsigned long long)(ms * 1e3);
        stats[12] = h2d;
        stats[13] = (unsigned long long)(n_shards * sizeof(SfShardOut) + n_reads * 8 + (out->elem_capacity > 0 ? n_elems * 17 : 0));
        stats[14] = (unsigned long long)launches;
    }
    return 0;
}
// =================================================================================================
// bank totals
// =================================================================================================
struct BkRead { int64_t pl_off; int32_t pl_len; int32_t index; };
struct BkAgg {
    unsigned long long count[5];
    int first_idx[5], last_idx[5];
    unsigned long long worst_key[5];   // orderable badness
    int worst_idx[5];
    long long lowest, highest;
    int lowest_idx, highest_idx;
    int first_error_idx;
    int pad;
};

__device__ __forceinline__ unsigned long long orderable(double d) {
    unsigned long long u = (unsigned long long)__double_as_longlong(d);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}

// pass 0: classify + value reductions; pass 1: arg-index resolution (first read attaining the extreme)
__global__ void bk_scan(const BkRead* __restrict__ reads, int64_t n_reads, const int32_t* __restrict__ payload,
                        int n_accounts, int4 acct_lo, int4 acct_hi, long long total_amount, int neg_ok, int pass,
                        uint8_t* __restrict__ type_out, BkAgg* __restrict__ agg) {
    const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    const BkRead rd = reads[r];
    const int ids[8] = {acct_lo.x, acct_lo.y, acct_lo.z, acct_lo.w, acct_hi.x, acct_hi.y, acct_hi.z, acct_hi.w};
    int n_unexpected = 0, n_nil = 0;
    long long total = 0, neg_sum = 0;
    bool any_neg = false;
    for (int i = 0; i + 1 < rd.pl_len; i += 2) {
        const int32_t id = __ldg(payload + rd.pl_off + i), bal = __ldg(payload + rd.pl_off + i + 1);
        bool known = false;
#pragma unroll
        for (int a = 0; a < 8; ++a) known |= a < n_accounts && ids[a] == id;
        n_unexpected += !known;
        if (bal == JTB_NIL) n_nil++;
        else { total += bal; if (bal < 0) { any_neg = true; neg_sum += bal; } }
    }
    int type = JTB_BANK_OK;
    if (n_unexpected) type = JTB_BANK_UNEXPECTED_KEY;
    else if (n_nil) type = JTB_BANK_NIL_BALANCE;
    else if (total != total_amount) type = JTB_BANK_WRONG_TOTAL;
    else if (!neg_ok && any_neg) type = JTB_BANK_NEGATIVE_VALUE;
    if (type == JTB_BANK_OK) { if (pass == 0) type_out[r] = 0; return; }
    double bad = 0;
    if (type == JTB_BANK_UNEXPECTED_KEY) bad = n_unexpected;
    else if (type == JTB_BANK_NIL_BALANCE) bad = n_nil;
    else if (type == JTB_BANK_WRONG_TOTAL)
        bad = total_amount == 0 ? fabs((double)(total - total_amount))
                                : fabs((double)(float)((double)(total - total_amount) / (double)total_amount));
    else bad = -(double)neg_sum;
    const unsigned long long bk = orderable(bad);
    if (pass == 0) {
        type_out[r] = (uint8_t)type;
        atomicAdd(&agg->count[type], 1ull);
        atomicMin(&agg->first_idx[type], rd.index);
        atomicMax(&agg->last_idx[type], rd.index);
        atomicMax(&agg->worst_key[type], bk);
        atomicMin(&agg->first_error_idx, rd.index);
        if (type == JTB_BANK_WRONG_TOTAL) { atomicMin(&agg->lowest, total); atomicMax(&agg->highest, total); }
    } else {
        if (agg->worst_key[type] == bk) atomicMin(&agg->worst_idx[type], rd.index);
        if (type == JTB_BANK_WRONG_TOTAL) {
            if (agg->lowest == total) atomicMin(&agg->lowest_idx, rd.index);
            if (agg->highest == total) atomicMin(&agg->highest_idx, rd.index);
        }
    }
}

inline int run_bank_totals(cudaStream_t st, cudaEvent_t e0, cudaEvent_t e1, const jtb_history* h, const jtb_model* m,
                           int64_t total_amount, jtb_bank_result* out, std::string& err) {
    const double t_start = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
    // zero accounts is legal (every key of every read is then unexpected); more than the model holds is not
    if (m->n_accounts < 0 || m->n_accounts > JTB_MAX_ACCOUNTS) { err = "bank model needs 0..8 accounts"; return -2; }
    std::vector<BkRead> reads;
    for (int64_t e = 0; e < h->n_events; ++e) {
        if (h->process[e] < 0 || h->type[e] != JTB_T_OK || h->f[e] != JTB_F_READ) continue;
        reads.push_back(BkRead{h->payload_off[e], std::max(0, (int)h->payload_len[e]), h->index[e]});
    }
    const int64_t n = (int64_t)reads.size();
    CallAllocs A;
    const BkRead* d_reads; const int32_t* d_payload; uint8_t* d_type; BkAgg* d_agg;
    JTB_OK(A.put(&d_reads, reads, st));
    JTB_OK(A.put(&d_payload, h->payload, (size_t)h->n_payload, st));
    JTB_OK(A.alloc(&d_type, (size_t)n));
    JTB_OK(A.alloc(&d_agg, 1));
    BkAgg init;
    std::memset(&init, 0, sizeof init);
    for (int t = 0; t < 5; ++t) { init.first_idx[t] = 0x7fffffff; init.last_idx[t] = -1; init.worst_idx[t] = 0x7fffffff; }
    init.lowest = INT64_MAX; init.highest = INT64_MIN;
    init.lowest_idx = init.highest_idx = init.first_error_idx = 0x7fffffff;
    JTB_OK(cudaMemcpyAsync(d_agg, &init, sizeof init, cudaMemcpyHostToDevice, st));
    int ids[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < m->n_accounts; ++i) ids[i] = m->account_ids[i];
    const int4 lo = make_int4(ids[0], ids[1], ids[2], ids[3]), hi = make_int4(ids[4], ids[5], ids[6], ids[7]);
    JTB_OK(cudaEventRecord(e0, st));
    if (n > 0) {
        for (int pass = 0; pass < 2; ++pass) {
            bk_scan<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_reads, n, d_payload, m->n_accounts, lo, hi, total_amount,
                                                                 m->negative_balances_ok, pass, d_type, d_agg);
            JTB_OK(cudaGetLastError());
        }
    }
    JTB_OK(cudaEventRecord(e1, st));
    BkAgg agg;
    JTB_OK(cudaMemcpyAsync(&agg, d_agg, sizeof agg, cudaMemcpyDeviceToHost, st));
    std::vector<uint8_t> types((size_t)n);
    JTB_OK(cudaMemcpyAsync(types.data(), d_type, n, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaStreamSynchronize(st));
    float ms = 0;
    JTB_OK(cudaEventElapsedTime(&ms, e0, e1));
    std::memset(out, 0, sizeof *out);
    out->read_count = n;
    out->first_error_index = -1;
    out->lowest_index = out->highest_index = -1;
    for (int t = 0; t < 5; ++t) {
        out->count_by_type[t] = (int64_t)agg.count[t];
        out->error_count += (t > 0) ? (int64_t)agg.count[t] : 0;
        out->first_index_by_type[t] = agg.count[t] ? agg.first_idx[t] : -1;
        out->last_index_by_type[t] = agg.count[t] ? agg.last_idx[t] : -1;
        out->worst_index_by_type[t] = agg.count[t] ? agg.worst_idx[t] : -1;
    }
    if (out->error_count) {
        out->first_error_index = agg.first_error_idx;
        for (int64_t r = 0; r < n; ++r)
            if (reads[r].index == agg.first_error_idx) { out->first_error_type = types[r]; break; }
    }
    if (agg.count[JTB_BANK_WRONG_TOTAL]) {
        out->lowest_total = agg.lowest; out->highest_total = agg.highest;
        out->lowest_index = agg.lowest_idx; out->highest_index = agg.highest_idx;
    }
    out->valid = out->error_count ? JTB_INVALID : JTB_VALID;
    // reference quirk (tests/ledger.clj:122-123 with the default :total-amount 0, :356): err-badness divides by zero as
    // soon as util/max-by has two :wrong-total errors to compare -> the checker throws -> check-safe: :unknown
    if (total_amount == 0 && agg.count[JTB_BANK_WRONG_TOTAL] >= 2) {
        out->reference_throws = 1;
        out->valid = JTB_UNKNOWN;
    }
    out->seconds_kernel = ms * 1e-3;
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count() - t_start;
    return 0;
}

}  // namespace jtb
