// jtb_call.cuh — the host side of one checker call that reports through `std::string& err`: the CUDA-error macro, the
// call's device allocations, input errors, the history prologue of the ledger checks and their result roll-up.
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/jtb_check.h"

// a failed CUDA call sets err to the call and its error and returns -1
#define JTB_OK(call)                                                                                      \
    do {                                                                                                  \
        cudaError_t e_ = (call);                                                                          \
        if (e_ != cudaSuccess) { err = std::string(#call) + ": " + cudaGetErrorString(e_); return -1; }  \
    } while (0)

namespace jtb {

// The device allocations of one call, released on every return path.  Every allocation has at least 16 bytes.  A
// refused cudaMalloc also stays behind as the thread's last error; it is cleared here, so that the next call's
// cudaGetLastError() check does not report it.
struct CallAllocs {
    std::vector<void*> ptrs;
    CallAllocs() = default;
    CallAllocs(const CallAllocs&) = delete;
    CallAllocs& operator=(const CallAllocs&) = delete;
    ~CallAllocs() { for (void* p : ptrs) cudaFree(p); }

    // n elements of T
    template <class T>
    cudaError_t alloc(T** p, size_t n) {
        void* q = nullptr;
        const cudaError_t e = cudaMalloc(&q, std::max<size_t>(n * sizeof(T), 16));
        if (e == cudaSuccess) ptrs.push_back(q);
        else (void)cudaGetLastError();
        *p = static_cast<T*>(q);
        return e;
    }
    // n elements of T, filled from src[0, n) on stream st (no copy when n = 0)
    template <class T>
    cudaError_t put(const T** p, const T* src, size_t n, cudaStream_t st) {
        T* q;
        cudaError_t e = alloc(&q, n);
        *p = q;
        if (e == cudaSuccess && n) e = cudaMemcpyAsync(q, src, n * sizeof(T), cudaMemcpyHostToDevice, st);
        return e;
    }
    template <class T>
    cudaError_t put(const T** p, const std::vector<T>& src, cudaStream_t st) {
        return put(p, src.data(), src.size(), st);
    }
};

// a malformed input: err = the formatted message, -2
__attribute__((format(printf, 2, 3))) inline int input_error(std::string& err, const char* fmt, ...) {
    char buf[256];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    err = buf;
    return -2;
}

// the arrays the ledger checks read are present (with transfers: also a, b and c) and the counts are not negative
inline int check_history(const jtb_history* h, bool transfers, std::string& err) {
    if (h->n_events < 0 || h->n_shards < 0 ||
        (h->n_events > 0 && (!h->type || !h->f || !h->process || !h->index || !h->payload_off || !h->payload_len ||
                             (transfers && (!h->a || !h->b || !h->c)))) ||
        !h->shard_off || (h->n_payload > 0 && !h->payload)) {
        err = "malformed jtb_history";
        return -2;
    }
    return 0;
}

// the call's verdict (the worst over its shards), its failures (the shards that are not VALID) and its two clocks
template <class Result, class Shard>
inline void roll_up(Result* out, const Shard* shards, int32_t n_shards, float ms_kernel,
                    std::chrono::steady_clock::time_point t0) {
    for (int32_t s = 0; s < n_shards; ++s) {
        out->valid = std::max(out->valid, shards[s].valid);
        if (shards[s].valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_kernel = ms_kernel * 1e-3;
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace jtb
