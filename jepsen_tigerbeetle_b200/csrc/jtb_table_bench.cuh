// jtb_table_bench.cuh — the visited-config table (K2) in isolation: insert + probe micro-benchmark used
// for the roofline evidence in DESIGN.md.  Keys are pseudo-random 128-bit values; the
// table is sized >> L2 (50 MB) so probes are honest HBM traffic.
//
// Probe variants:
//   0  slot probing     one lane per key, ld.global.cg.v2.u64 of the 16 B home slot, linear probing
//                       (this is the path the search kernel uses)
//   1  bucket / LDG     8 lanes cooperate on one key: one coalesced 128 B bucket read (8 x 16 B),
//                       match by ballot
//   2  bucket / TMA     one lane per key issues cp.async.bulk (global -> shared, 128 B) with an
//                       mbarrier; buckets are then scanned in shared memory
// Variants 1 and 2 use a bucketed layout (home bucket = hash, slot = first empty in the bucket).
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>

#include "jtb_wgl.cuh"

namespace jtb {

__device__ __forceinline__ void bench_key(uint64_t i, uint64_t (&k)[2]) {
    k[0] = mix64(i * 2 + 1) | KEY_VALID;
    k[0] &= ~KEY_LOCK;
    k[1] = mix64(i * 2 + 2);
}

__global__ void tb_insert_slots(uint64_t* table, uint64_t slot_mask, uint64_t n_keys, unsigned long long* inserted) {
    unsigned long long mine = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_keys; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t k[2];
        bench_key(i, k);
        int plen;
        mine += table_insert<2>(table, slot_mask, k, &plen) > 0;
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(inserted, mine);
}

__global__ void tb_insert_buckets(uint64_t* table, uint64_t bucket_mask, uint64_t n_keys, unsigned long long* inserted) {
    unsigned long long mine = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_keys; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t k[2];
        bench_key(i, k);
        uint64_t b = hash_key<2>(k) & bucket_mask;
        bool done = false;
        for (int tries = 0; tries < 64 && !done; ++tries) {
            for (int s = 0; s < 8 && !done; ++s) {
                uint64_t* slot = table + (b * 8 + s) * 2;
                K128 cur = ldcg128(slot);
                if (cur.lo == 0 && cur.hi == 0) cur = cas128(slot, K128{0, 0}, K128{k[0], k[1]});
                else if (cur.lo == k[0] && cur.hi == k[1]) { done = true; break; }
                else continue;
                if (cur.lo == 0 && cur.hi == 0) { done = true; mine++; }
                else if (cur.lo == k[0] && cur.hi == k[1]) done = true;
            }
            b = (b + 1) & bucket_mask;
        }
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(inserted, mine);
}

// variant 0: 4 independent probes in flight per lane
__global__ void __launch_bounds__(256) tb_probe_slots(const uint64_t* table, uint64_t slot_mask, uint64_t n_keys,
                                                      uint64_t salt, unsigned long long* found) {
    unsigned long long mine = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i0 < n_keys; i0 += 4 * stride) {
        uint64_t k[4][2], idx[4];
        K128 cur[4];
        bool live[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint64_t i = i0 + u * stride;
            live[u] = i < n_keys;
            bench_key((i + salt) % n_keys, k[u]);
            idx[u] = hash_key<2>(k[u]) & slot_mask;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (live[u]) cur[u] = ldcg128(table + idx[u] * 2);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (!live[u]) continue;
            for (int p = 0; p < MAX_PROBE; ++p) {
                if (cur[u].lo == k[u][0] && cur[u].hi == k[u][1]) { mine++; break; }
                if (cur[u].lo == 0 && cur[u].hi == 0) break;
                idx[u] = (idx[u] + 1) & slot_mask;
                cur[u] = ldcg128(table + idx[u] * 2);
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(found, mine);
}

// variant 1: 8 lanes per key, one coalesced 128 B bucket load
__global__ void __launch_bounds__(256) tb_probe_buckets_ldg(const uint64_t* table, uint64_t bucket_mask, uint64_t n_keys,
                                                            uint64_t salt, unsigned long long* found) {
    unsigned long long mine = 0;
    const int sub = threadIdx.x & 7;
    const uint64_t group = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 3;
    const uint64_t n_groups = ((uint64_t)gridDim.x * blockDim.x) >> 3;
    for (uint64_t i0 = group; i0 < n_keys; i0 += 4 * n_groups) {
        uint64_t k[4][2], b[4];
        K128 cur[4];
        bool live[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint64_t i = i0 + u * n_groups;
            live[u] = i < n_keys;
            bench_key((i + salt) % n_keys, k[u]);
            b[u] = hash_key<2>(k[u]) & bucket_mask;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (live[u]) cur[u] = ldcg128(table + (b[u] * 8 + sub) * 2);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            for (int tries = 0; tries < 64; ++tries) {
                const bool hit = live[u] && cur[u].lo == k[u][0] && cur[u].hi == k[u][1];
                const bool empty = live[u] && cur[u].lo == 0 && cur[u].hi == 0;
                const unsigned gm = 0xffu << ((threadIdx.x & 31) & ~7);  // the 8 lanes sharing this key
                const unsigned hits = __ballot_sync(gm, hit);
                const unsigned empties = __ballot_sync(gm, empty);
                if (hits) { if (sub == 0) mine++; break; }
                if (empties || !live[u]) break;
                b[u] = (b[u] + 1) & bucket_mask;
                cur[u] = ldcg128(table + (b[u] * 8 + sub) * 2);
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(found, mine);
}

// variant 2: cp.async.bulk staging of 128 B buckets into shared memory, one mbarrier per warp
__global__ void __launch_bounds__(128) tb_probe_buckets_tma(const uint64_t* table, uint64_t bucket_mask, uint64_t n_keys,
                                                            uint64_t salt, unsigned long long* found) {
    __shared__ __align__(128) uint8_t stage[4][2][32 * 128];  // per warp, double buffered
    __shared__ __align__(8) uint64_t bars[4][2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) {
        for (int s = 0; s < 2; ++s) {
            const uint32_t a = (uint32_t)__cvta_generic_to_shared(&bars[warp][s]);
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(1));
        }
        asm volatile("fence.mbarrier_init.release.cluster;");
    }
    __syncwarp();
    unsigned long long mine = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    uint32_t phase[2] = {0, 0};
    uint64_t kcur[2][2];
    bool livecur[2] = {false, false};
    auto issue = [&](int s, uint64_t ii) {
        livecur[s] = ii < n_keys;
        bench_key((ii + salt) % n_keys, kcur[s]);
        const uint64_t b = hash_key<2>(kcur[s]) & bucket_mask;
        const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[warp][s]);
        const unsigned lm = __ballot_sync(0xffffffffu, livecur[s]);
        if (lane == 0 && lm)
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(128 * __popc(lm)) : "memory");
        __syncwarp();
        if (livecur[s]) {
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(&stage[warp][s][lane * 128]);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst), "l"(table + b * 16), "r"(128), "r"(bar) : "memory");
        }
        return lm;
    };
    unsigned lm_cur = issue(0, i);
    int s = 0;
    while (lm_cur) {
        const unsigned lm_next = issue(s ^ 1, i + stride);
        // wait for stage s
        const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[warp][s]);
        uint32_t ok = 0;
        while (!ok)
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(ok) : "r"(bar), "r"(phase[s]) : "memory");
        phase[s] ^= 1;
        if (livecur[s]) {
            const K128* bk = reinterpret_cast<const K128*>(&stage[warp][s][lane * 128]);
            bool hit = false;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const K128 c = bk[(q + lane) & 7];  // rotate start slot: conflict-free across lanes
                hit |= c.lo == kcur[s][0] && c.hi == kcur[s][1];
            }
            mine += hit;  // (overflow buckets are ignored by this variant: load factor kept low)
        }
        __syncwarp();
        i += stride;
        s ^= 1;
        lm_cur = lm_next;
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if (lane == 0) atomicAdd(found, mine);
}

// ---- random-gather sweep: what the memory system gives a hash probe, as a function of the table's footprint ----------
// Every thread walks its own pseudo-random slot sequence (xorshift32 + one multiply: the address generation costs a
// handful of instructions, so the ALUs are not what is measured) with U independent 16 B loads (ld.global.cg.v2.u64,
// exactly the search kernel's probe) in flight; WIDE = 2 also loads the other half of the 32 B sector.  The loaded
// words are folded into a checksum so nothing is optimised away.  Footprints from a few MiB (inside the 50 MB L2) to
// 16 GiB show where random 16 B probes stop being served by L2 and what DRAM / the TLBs sustain beyond it.
template <int U, int WIDE>
__global__ void __launch_bounds__(256) tb_gather(const uint64_t* __restrict__ table, uint64_t slot_mask, uint32_t iters,
                                                 unsigned long long* sink) {
    uint32_t x = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u + 12345u;
    uint64_t acc = 0;
    for (uint32_t it = 0; it < iters; ++it) {
        K128 v[U], w[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            x ^= x << 13; x ^= x >> 17; x ^= x << 5;
            const uint64_t idx = ((uint64_t)x * 0x9E3779B97F4A7C15ull >> 20) & slot_mask;
            v[u] = ldcg128(table + idx * 2);
            if (WIDE == 2) w[u] = ldcg128(table + (idx ^ 1) * 2);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            acc ^= v[u].lo + v[u].hi;
            if (WIDE == 2) acc ^= w[u].lo + w[u].hi;
        }
    }
    if (acc == 0x123456789abcdefull) atomicAdd(sink, 1ull);   // never true in practice: keeps the loads alive
}

template <int U, int WIDE>
int launch_gather(cudaStream_t st, const uint64_t* table, uint64_t slot_mask, uint32_t iters, int grid,
                  unsigned long long* sink) {
    tb_gather<U, WIDE><<<grid, 256, 0, st>>>(table, slot_mask, iters, sink);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// loads = grid * 256 * iters * U probes of 16 B (x WIDE); returns seconds (CUDA events), best of `rounds`
inline int run_gather_bench(cudaStream_t st, cudaEvent_t e0, cudaEvent_t e1, uint64_t* table, uint64_t n_slots, int in_flight,
                            int wide, uint32_t iters, int ctas_per_sm, int rounds, int n_sms, double* seconds,
                            uint64_t* n_probes, std::string& err) {
    unsigned long long* d_sink = nullptr;
    if (cudaMalloc(&d_sink, 8) != cudaSuccess) { err = "cudaMalloc failed"; return -1; }
    cudaMemsetAsync(d_sink, 0, 8, st);
    // non-zero contents (an all-zero table could be served by compression / zero pages)
    if (cudaMemsetAsync(table, 0x5a, n_slots * 16, st) != cudaSuccess) { err = "memset failed"; cudaFree(d_sink); return -1; }
    const int grid = n_sms * ctas_per_sm;
    double best = 1e30;
    for (int r = 0; r < rounds + 1; ++r) {   // first round = warm-up
        cudaEventRecord(e0, st);
        int rc = -1;
        const uint64_t mask = n_slots - 1;
#define JTB_G(U_, W_) rc = launch_gather<U_, W_>(st, table, mask, iters, grid, d_sink)
        if (wide == 2) { if (in_flight <= 2) JTB_G(2, 2); else if (in_flight <= 4) JTB_G(4, 2); else if (in_flight <= 8) JTB_G(8, 2); else JTB_G(16, 2); }
        else { if (in_flight <= 1) JTB_G(1, 1); else if (in_flight <= 2) JTB_G(2, 1); else if (in_flight <= 4) JTB_G(4, 1); else if (in_flight <= 8) JTB_G(8, 1); else JTB_G(16, 1); }
#undef JTB_G
        cudaEventRecord(e1, st);
        if (rc || cudaStreamSynchronize(st) != cudaSuccess) { err = "gather kernel failed"; cudaFree(d_sink); return -1; }
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        if (r > 0) best = std::min(best, (double)ms * 1e-3);
    }
    cudaFree(d_sink);
    const int u = in_flight <= 1 ? 1 : in_flight <= 2 ? 2 : in_flight <= 4 ? 4 : in_flight <= 8 ? 8 : 16;
    *seconds = best;
    *n_probes = (uint64_t)grid * 256ull * iters * (uint64_t)(wide == 2 && u < 2 ? 2 : u);
    return 0;
}

inline int run_table_bench(cudaStream_t st, cudaEvent_t e0, cudaEvent_t e1, uint64_t* table, uint64_t n_slots,
                           uint64_t n_keys, int variant, int rounds, int n_sms, double* ins_s, double* probe_s,
                           uint64_t* found, std::string& err) {
    auto fail = [&](cudaError_t e, const char* what) {
        err = std::string(what) + ": " + cudaGetErrorString(e);
        return -1;
    };
    cudaError_t e;
    unsigned long long* d_cnt = nullptr;
    if ((e = cudaMalloc(&d_cnt, 16)) != cudaSuccess) return fail(e, "cudaMalloc");
    if ((e = cudaMemsetAsync(table, 0, n_slots * 16, st)) != cudaSuccess) return fail(e, "memset");
    cudaMemsetAsync(d_cnt, 0, 16, st);
    const int grid = n_sms * 8;
    cudaEventRecord(e0, st);
    if (variant == 0) tb_insert_slots<<<grid, 256, 0, st>>>(table, n_slots - 1, n_keys, d_cnt);
    else tb_insert_buckets<<<grid, 256, 0, st>>>(table, n_slots / 8 - 1, n_keys, d_cnt);
    cudaEventRecord(e1, st);
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return fail(e, "insert kernel");
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    *ins_s = ms * 1e-3;
    cudaEventRecord(e0, st);
    for (int r = 0; r < rounds; ++r) {
        const uint64_t salt = 0x9E3779B9ull * (r + 1);
        if (variant == 0) tb_probe_slots<<<grid, 256, 0, st>>>(table, n_slots - 1, n_keys, salt, d_cnt + 1);
        else if (variant == 1) tb_probe_buckets_ldg<<<grid, 256, 0, st>>>(table, n_slots / 8 - 1, n_keys, salt, d_cnt + 1);
        else tb_probe_buckets_tma<<<grid * 2, 128, 0, st>>>(table, n_slots / 8 - 1, n_keys, salt, d_cnt + 1);
    }
    cudaEventRecord(e1, st);
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return fail(e, "probe kernel");
    cudaEventElapsedTime(&ms, e0, e1);
    *probe_s = ms * 1e-3;
    unsigned long long h[2];
    cudaMemcpy(h, d_cnt, 16, cudaMemcpyDeviceToHost);
    cudaFree(d_cnt);
    *found = h[1];
    return 0;
}

}  // namespace jtb
