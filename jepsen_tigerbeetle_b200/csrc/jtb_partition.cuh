// jtb_partition.cuh — SURVEY §8(f) N2: the step immediately BEFORE the checkers, on the device.
//
//  * jepsen.independent/subhistory (set_full.clj:155: `independent/checker` re-filters the whole history once per key,
//    O(keys x events)): ONE stable partition of the events by key — radix sort of (key, event index) pairs (cub), then
//    the run boundaries give the CSR `shard_off` / `key_ids` of `jtb_history`.  `order[i]` = original position of the
//    i-th event of the partitioned history; events of one key keep their history order (stable sort).
//  * ledger->bank (tests/ledger.clj:100-105): a read's `{:credits-posted c :debits-posted d}` -> balance c - d, elementwise.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <cub/cub.cuh>
#include <cuda_runtime.h>

#include "jtb_call.cuh"

namespace jtb {

__global__ void pt_init(const int64_t* __restrict__ key, int64_t n, uint64_t* __restrict__ k, int32_t* __restrict__ idx) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) { k[i] = (uint64_t)key[i] ^ 0x8000000000000000ull; idx[i] = (int32_t)i; }   // signed order as unsigned
}
// heads[i] = 1 where a new key starts; run index by prefix sum (cub) -> offsets
__global__ void pt_heads(const uint64_t* __restrict__ k, int64_t n, int32_t* __restrict__ head) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) head[i] = (i == 0 || k[i] != k[i - 1]) ? 1 : 0;
}
__global__ void pt_emit(const uint64_t* __restrict__ k, const int32_t* __restrict__ head, const int32_t* __restrict__ run,
                        int64_t n, int64_t* __restrict__ shard_off, int64_t* __restrict__ key_ids, int32_t cap) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n && head[i]) {
        const int32_t r = run[i] - 1;   // inclusive scan: 1-based
        if (r < cap) { shard_off[r] = i; key_ids[r] = (int64_t)(k[i] ^ 0x8000000000000000ull); }
    }
}
__global__ void pt_balances(const int64_t* __restrict__ credits, const int64_t* __restrict__ debits, int64_t n, int32_t* __restrict__ out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = (int32_t)(credits[i] - debits[i]);
}

inline int run_partition_by_key(cudaStream_t st, int64_t n, const int64_t* event_key, int32_t* order, int64_t* shard_off,
                                int64_t* key_ids, int32_t key_cap, int32_t* n_keys, std::string& err) {
    *n_keys = 0;
    if (n <= 0) { if (key_cap >= 0) shard_off[0] = 0; return 0; }
    if (n >= (1ll << 31)) { err = "too many events"; return -2; }
    const unsigned grid = (unsigned)((n + 255) / 256);
    CallAllocs A;
    const int64_t* d_key;
    uint64_t *d_k0, *d_k1;
    int32_t *d_i0, *d_i1, *d_head, *d_run;
    int64_t *d_off, *d_ids;
    uint8_t* d_tmp;
    JTB_OK(A.put(&d_key, event_key, (size_t)n, st)); JTB_OK(A.alloc(&d_k0, n)); JTB_OK(A.alloc(&d_k1, n));
    JTB_OK(A.alloc(&d_i0, n)); JTB_OK(A.alloc(&d_i1, n)); JTB_OK(A.alloc(&d_head, n)); JTB_OK(A.alloc(&d_run, n));
    JTB_OK(A.alloc(&d_off, (size_t)key_cap + 1)); JTB_OK(A.alloc(&d_ids, (size_t)key_cap + 1));
    pt_init<<<grid, 256, 0, st>>>(d_key, n, d_k0, d_i0);
    size_t tmp_sort = 0, tmp_scan = 0;
    JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, (const uint64_t*)d_k0, d_k1, (const int32_t*)d_i0, d_i1, (int)n, 0, 64, st));
    JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, tmp_scan, (const int32_t*)d_head, d_run, (int)n, st));
    JTB_OK(A.alloc(&d_tmp, std::max(tmp_sort, tmp_scan)));
    size_t tb = std::max(tmp_sort, tmp_scan);
    JTB_OK(cub::DeviceRadixSort::SortPairs(d_tmp, tb, (const uint64_t*)d_k0, d_k1, (const int32_t*)d_i0, d_i1, (int)n, 0, 64, st));
    pt_heads<<<grid, 256, 0, st>>>(d_k1, n, d_head);
    tb = std::max(tmp_sort, tmp_scan);
    JTB_OK(cub::DeviceScan::InclusiveSum(d_tmp, tb, (const int32_t*)d_head, d_run, (int)n, st));
    pt_emit<<<grid, 256, 0, st>>>(d_k1, d_head, d_run, n, d_off, d_ids, key_cap);
    JTB_OK(cudaGetLastError());
    int32_t total = 0;
    JTB_OK(cudaMemcpyAsync(&total, d_run + (n - 1), 4, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaMemcpyAsync(order, d_i1, n * 4, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaStreamSynchronize(st));
    if (total > key_cap) { err = "key_cap too small"; return -4; }
    JTB_OK(cudaMemcpy(shard_off, d_off, (size_t)total * 8, cudaMemcpyDeviceToHost));
    JTB_OK(cudaMemcpy(key_ids, d_ids, (size_t)total * 8, cudaMemcpyDeviceToHost));
    shard_off[total] = n;
    *n_keys = total;
    return 0;
}

inline int run_ledger_balances(cudaStream_t st, int64_t n, const int64_t* credits, const int64_t* debits, int32_t* out, std::string& err) {
    if (n <= 0) return 0;
    CallAllocs A;
    const int64_t *d_c, *d_d;
    int32_t* d_o;
    JTB_OK(A.put(&d_c, credits, (size_t)n, st)); JTB_OK(A.put(&d_d, debits, (size_t)n, st)); JTB_OK(A.alloc(&d_o, n));
    pt_balances<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_c, d_d, n, d_o);
    JTB_OK(cudaGetLastError());
    JTB_OK(cudaMemcpyAsync(out, d_o, n * 4, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaStreamSynchronize(st));
    return 0;
}

}  // namespace jtb
