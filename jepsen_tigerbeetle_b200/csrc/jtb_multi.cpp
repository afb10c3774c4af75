// jtb_multi.cpp — multi-GPU fan-out inside the library (include/jtb_check.h, "jtb_multi_*").
//
// The multi-GPU shape of `independent/checker` (src/tigerbeetle/workloads/set_full.clj:155) for a single-process host
// (a JVM through JNI): shards = independent keys, partitioned over the devices of the box by LPT on events^2, one
// host thread and one jtb_ctx per device, no configuration ever crosses GPUs.  The only collective is ONE
// ncclAllReduce(ncclMax) over int32[3 * n_shards] — (verdict, witness :index, previous-ok :index) per shard, verdict
// codes ordered like jepsen.checker/merge-valid (true 0 < :unknown 1 < false 2) — over NVLink/NVSwitch.
// NCCL is dlopen'ed here: libjtb_check.so has no link-time dependency on it.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <numeric>
#include <string>
#include <thread>
#include <vector>

#include "../../include/jtb_check.h"

namespace {

struct NcclApi {
    void* handle = nullptr;
    decltype(&ncclCommInitAll) CommInitAll = nullptr;
    decltype(&ncclCommDestroy) CommDestroy = nullptr;
    decltype(&ncclAllReduce) AllReduce = nullptr;
    decltype(&ncclGroupStart) GroupStart = nullptr;
    decltype(&ncclGroupEnd) GroupEnd = nullptr;
    decltype(&ncclGetErrorString) GetErrorString = nullptr;
    bool load(std::string& err) {
        for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
            handle = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
            if (handle) break;
        }
        if (!handle) { err = std::string("NCCL not found: ") + dlerror(); return false; }
#define JTB_SYM(f)                                                        \
    f = reinterpret_cast<decltype(f)>(dlsym(handle, "nccl" #f));          \
    if (!f) { err = "NCCL symbol missing: nccl" #f; return false; }
        JTB_SYM(CommInitAll) JTB_SYM(CommDestroy) JTB_SYM(AllReduce) JTB_SYM(GroupStart) JTB_SYM(GroupEnd)
        JTB_SYM(GetErrorString)
#undef JTB_SYM
        return true;
    }
};

std::string g_create_err;
std::mutex g_create_mu;

// A subset of the shards of `h` as a history of its own (arrays owned here; the payload is compacted so that a
// device only ever uploads the id lists / balances of its own shards).
struct SubHistory {
    std::vector<uint8_t> type, f, flags;
    std::vector<int32_t> process, index, a, b, c, payload_len, payload;
    std::vector<int64_t> time_ns, payload_off, shard_off, key_ids;
    jtb_history h{};
    void build(const jtb_history* src, const std::vector<int>& shards) {
        int64_t n = 0, np = 0;
        for (int s : shards) {
            n += src->shard_off[s + 1] - src->shard_off[s];
            for (int64_t e = src->shard_off[s]; e < src->shard_off[s + 1]; ++e) np += std::max(0, src->payload_len[e]);
        }
        type.resize(n); f.resize(n); flags.assign(n, 0); process.resize(n); index.resize(n); a.resize(n); b.resize(n);
        c.resize(n); payload_len.resize(n); time_ns.resize(n); payload_off.resize(n); payload.resize(np);
        shard_off.assign(1, 0);
        key_ids.clear();
        int64_t o = 0, po = 0;
        for (int s : shards) {
            const int64_t lo = src->shard_off[s], cnt = src->shard_off[s + 1] - lo;
            std::memcpy(type.data() + o, src->type + lo, cnt);
            std::memcpy(f.data() + o, src->f + lo, cnt);
            if (src->flags) std::memcpy(flags.data() + o, src->flags + lo, cnt);
            std::memcpy(process.data() + o, src->process + lo, cnt * 4);
            std::memcpy(index.data() + o, src->index + lo, cnt * 4);
            std::memcpy(a.data() + o, src->a + lo, cnt * 4);
            std::memcpy(b.data() + o, src->b + lo, cnt * 4);
            std::memcpy(c.data() + o, src->c + lo, cnt * 4);
            std::memcpy(payload_len.data() + o, src->payload_len + lo, cnt * 4);
            std::memcpy(time_ns.data() + o, src->time_ns + lo, cnt * 8);
            for (int64_t e = 0; e < cnt; ++e) {
                const int len = std::max(0, src->payload_len[lo + e]);
                payload_off[o + e] = po;
                if (len) std::memcpy(payload.data() + po, src->payload + src->payload_off[lo + e], (size_t)len * 4);
                po += len;
            }
            o += cnt;
            shard_off.push_back(o);
            key_ids.push_back(src->key_ids ? src->key_ids[s] : (int64_t)s);
        }
        h.n_events = n;
        h.type = type.data(); h.f = f.data(); h.flags = flags.data(); h.process = process.data();
        h.index = index.data(); h.time_ns = time_ns.data(); h.a = a.data(); h.b = b.data(); h.c = c.data();
        h.payload_off = payload_off.data(); h.payload_len = payload_len.data(); h.payload = payload.data();
        h.n_payload = np;
        h.n_shards = (int32_t)shards.size();
        h.shard_off = shard_off.data();
        h.key_ids = key_ids.data();
    }
};

double now_s() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

}  // namespace

struct jtb_multi {
    int n = 0;
    std::vector<jtb_ctx*> ctx;
    std::vector<ncclComm_t> comms;
    std::vector<cudaStream_t> streams;
    std::vector<int32_t*> d_vec;     // per device: int32[vec_cap]
    size_t vec_cap = 0;
    NcclApi nccl;
    std::string err;
    std::mutex mu;
};

namespace {

// longest-processing-time-first partition of the shards over the devices (deterministic; cost = events^2)
std::vector<std::vector<int>> partition(const jtb_history* h, int n_dev) {
    std::vector<int> order(h->n_shards);
    std::iota(order.begin(), order.end(), 0);
    auto cost = [&](int s) { const double e = (double)(h->shard_off[s + 1] - h->shard_off[s]); return e * e; };
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return cost(x) > cost(y); });
    std::vector<double> load(n_dev, 0.0);
    std::vector<std::vector<int>> out(n_dev);
    for (int s : order) {
        const int d = (int)(std::min_element(load.begin(), load.end()) - load.begin());
        out[d].push_back(s);
        load[d] += cost(s);
    }
    for (auto& v : out) std::sort(v.begin(), v.end());
    return out;
}

// element-wise MAX of every device's int32 vector, through NCCL; `host` gets device 0's copy of the result
int merge_max(jtb_multi* mg, const std::vector<std::vector<int32_t>>& mine, std::vector<int32_t>& host) {
    const size_t count = host.size();
    if (count > mg->vec_cap) {
        for (int d = 0; d < mg->n; ++d) {
            cudaSetDevice(d);
            if (mg->d_vec[d]) cudaFree(mg->d_vec[d]);
            mg->d_vec[d] = nullptr;
            if (cudaMalloc(&mg->d_vec[d], count * 4) != cudaSuccess) { mg->err = "cudaMalloc (verdict vector) failed"; return -1; }
        }
        mg->vec_cap = count;
    }
    for (int d = 0; d < mg->n; ++d) {
        cudaSetDevice(d);
        if (cudaMemcpyAsync(mg->d_vec[d], mine[d].data(), count * 4, cudaMemcpyHostToDevice, mg->streams[d]) != cudaSuccess) {
            mg->err = "H2D of the verdict vector failed";
            return -1;
        }
    }
    ncclResult_t rc = mg->nccl.GroupStart();
    for (int d = 0; d < mg->n && rc == ncclSuccess; ++d)
        rc = mg->nccl.AllReduce(mg->d_vec[d], mg->d_vec[d], count, ncclInt32, ncclMax, mg->comms[d], mg->streams[d]);
    const ncclResult_t rc2 = mg->nccl.GroupEnd();
    if (rc == ncclSuccess) rc = rc2;
    if (rc != ncclSuccess) { mg->err = std::string("ncclAllReduce: ") + mg->nccl.GetErrorString(rc); return -1; }
    for (int d = 0; d < mg->n; ++d) {
        cudaSetDevice(d);
        if (d == 0) cudaMemcpyAsync(host.data(), mg->d_vec[0], count * 4, cudaMemcpyDeviceToHost, mg->streams[0]);
        if (cudaStreamSynchronize(mg->streams[d]) != cudaSuccess) { mg->err = "verdict all-reduce failed on the device"; return -1; }
    }
    return 0;
}

}  // namespace

extern "C" {

const char* jtb_multi_create_error(void) {
    std::lock_guard<std::mutex> lk(g_create_mu);
    return g_create_err.c_str();
}

jtb_multi* jtb_multi_create(const jtb_opts* opts, int n_gpus) {
    std::lock_guard<std::mutex> lk(g_create_mu);
    g_create_err.clear();
    const int avail = jtb_device_count();
    if (avail <= 0) { g_create_err = "no CUDA device (there is no CPU fallback)"; return nullptr; }
    if (n_gpus <= 0) n_gpus = avail;
    if (n_gpus > avail) { g_create_err = "more GPUs requested than visible"; return nullptr; }
    jtb_multi* mg = new jtb_multi();
    mg->n = n_gpus;
    auto fail = [&](const std::string& why) -> jtb_multi* {
        g_create_err = why;
        jtb_multi_destroy(mg);
        return nullptr;
    };
    if (!mg->nccl.load(g_create_err)) { const std::string e = g_create_err; return fail(e); }
    mg->ctx.assign(n_gpus, nullptr);
    mg->streams.assign(n_gpus, nullptr);
    mg->d_vec.assign(n_gpus, nullptr);
    for (int d = 0; d < n_gpus; ++d) {
        jtb_opts o{};
        if (opts) o = *opts;
        o.device = d;
        mg->ctx[d] = jtb_create(&o);
        if (!mg->ctx[d]) return fail("jtb_create failed on device " + std::to_string(d));
        cudaSetDevice(d);
        if (cudaStreamCreateWithFlags(&mg->streams[d], cudaStreamNonBlocking) != cudaSuccess) return fail("cudaStreamCreate failed");
    }
    mg->comms.assign(n_gpus, nullptr);
    std::vector<int> devs(n_gpus);
    std::iota(devs.begin(), devs.end(), 0);
    const ncclResult_t rc = mg->nccl.CommInitAll(mg->comms.data(), n_gpus, devs.data());
    if (rc != ncclSuccess) {
        mg->comms.clear();
        return fail(std::string("ncclCommInitAll: ") + mg->nccl.GetErrorString(rc));
    }
    return mg;
}

void jtb_multi_destroy(jtb_multi* mg) {
    if (!mg) return;
    for (size_t d = 0; d < mg->comms.size(); ++d)
        if (mg->comms[d]) mg->nccl.CommDestroy(mg->comms[d]);
    for (int d = 0; d < (int)mg->ctx.size(); ++d) {
        cudaSetDevice(d);
        if (d < (int)mg->d_vec.size() && mg->d_vec[d]) cudaFree(mg->d_vec[d]);
        if (d < (int)mg->streams.size() && mg->streams[d]) cudaStreamDestroy(mg->streams[d]);
        if (mg->ctx[d]) jtb_destroy(mg->ctx[d]);
    }
    delete mg;
}

int jtb_multi_n_gpus(const jtb_multi* mg) { return mg ? mg->n : 0; }
const char* jtb_multi_last_error(const jtb_multi* mg) { return mg ? mg->err.c_str() : "no multi-GPU context"; }

int jtb_multi_check_linearizable(jtb_multi* mg, const jtb_history* h, const jtb_model* m, jtb_lin_shard* shards,
                                 jtb_lin_result* out, int32_t* device_of_shard) {
    if (!mg) return -1;
    std::lock_guard<std::mutex> lk(mg->mu);
    const double t0 = now_s();
    const int ns = h->n_shards, nd = mg->n;
    const auto parts = partition(h, nd);
    std::vector<std::vector<jtb_lin_shard>> sub_shards(nd);
    std::vector<jtb_lin_result> sub_out(nd);
    std::vector<int> rcs(nd, 0);
    std::vector<std::string> errs(nd);
    std::vector<std::vector<int32_t>> mine(nd, std::vector<int32_t>((size_t)3 * ns, -1));
    std::vector<std::thread> th;
    for (int d = 0; d < nd; ++d) {
        std::memset(&sub_out[d], 0, sizeof sub_out[d]);
        if (parts[d].empty()) continue;
        th.emplace_back([&, d]() {
            SubHistory sub;
            sub.build(h, parts[d]);
            sub_shards[d].resize(parts[d].size());
            rcs[d] = jtb_check_linearizable(mg->ctx[d], &sub.h, m, sub_shards[d].data(), &sub_out[d]);
            if (rcs[d]) { errs[d] = jtb_last_error(mg->ctx[d]); return; }
            for (size_t k = 0; k < parts[d].size(); ++k) {
                const int s = parts[d][k];
                mine[d][s] = sub_shards[d][k].valid;
                mine[d][ns + s] = sub_shards[d][k].witness_index;
                mine[d][2 * ns + s] = sub_shards[d][k].previous_ok_index;
            }
        });
    }
    for (auto& t : th) t.join();
    for (int d = 0; d < nd; ++d)
        if (rcs[d]) { mg->err = "device " + std::to_string(d) + ": " + errs[d]; return rcs[d]; }
    std::vector<int32_t> merged((size_t)3 * ns, -1);
    if (ns > 0 && merge_max(mg, mine, merged)) return -1;
    std::memset(out, 0, sizeof *out);
    for (int d = 0; d < nd; ++d) {
        for (size_t k = 0; k < parts[d].size(); ++k) {
            const int s = parts[d][k];
            shards[s] = sub_shards[d][k];                 // cause, configs, probes: host-side detail
            shards[s].valid = merged[s];                  // verdict / witness: what came back over NVLink
            shards[s].witness_index = merged[ns + s];
            shards[s].previous_ok_index = merged[2 * ns + s];
            if (device_of_shard) device_of_shard[s] = d;
        }
        out->configs_explored += sub_out[d].configs_explored;
        out->probes += sub_out[d].probes;
        out->hbm_bytes_algorithmic += sub_out[d].hbm_bytes_algorithmic;
        out->key_bytes = std::max(out->key_bytes, sub_out[d].key_bytes);
        out->seconds_kernel = std::max(out->seconds_kernel, sub_out[d].seconds_kernel);
    }
    for (int s = 0; s < ns; ++s) {
        out->valid = std::max(out->valid, shards[s].valid);
        out->n_failures += shards[s].valid != JTB_VALID;
    }
    out->seconds_total = now_s() - t0;
    return 0;
}

int jtb_multi_check_set_full(jtb_multi* mg, const jtb_history* h, int linearizable, jtb_setfull_out* out,
                             int32_t* device_of_shard) {
    if (!mg) return -1;
    std::lock_guard<std::mutex> lk(mg->mu);
    if (out->elem_capacity || out->suspect_capacity || out->missing_capacity) {
        mg->err = "jtb_multi_check_set_full merges the per-shard structs only: unset the detail capacities";
        return -2;
    }
    const double t0 = now_s();
    const int ns = h->n_shards, nd = mg->n;
    const auto parts = partition(h, nd);
    std::vector<std::vector<jtb_setfull_shard>> sub_shards(nd);
    std::vector<jtb_setfull_out> sub_out(nd);
    std::vector<int> rcs(nd, 0);
    std::vector<std::string> errs(nd);
    std::vector<std::vector<int32_t>> mine(nd, std::vector<int32_t>((size_t)ns, -1));
    std::vector<std::thread> th;
    for (int d = 0; d < nd; ++d) {
        std::memset(&sub_out[d], 0, sizeof sub_out[d]);
        if (parts[d].empty()) continue;
        th.emplace_back([&, d]() {
            SubHistory sub;
            sub.build(h, parts[d]);
            sub_shards[d].resize(parts[d].size());
            sub_out[d].shards = sub_shards[d].data();
            rcs[d] = jtb_check_set_full(mg->ctx[d], &sub.h, linearizable, &sub_out[d]);
            if (rcs[d]) { errs[d] = jtb_last_error(mg->ctx[d]); return; }
            for (size_t k = 0; k < parts[d].size(); ++k) mine[d][parts[d][k]] = sub_shards[d][k].valid;
        });
    }
    for (auto& t : th) t.join();
    for (int d = 0; d < nd; ++d)
        if (rcs[d]) { mg->err = "device " + std::to_string(d) + ": " + errs[d]; return rcs[d]; }
    std::vector<int32_t> merged((size_t)ns, -1);
    if (ns > 0 && merge_max(mg, mine, merged)) return -1;
    out->valid = JTB_VALID;
    out->n_failures = 0;
    out->n_suspect = 0;
    out->raia_valid = JTB_VALID;
    out->seconds_kernel = 0;
    for (int d = 0; d < nd; ++d) {
        for (size_t k = 0; k < parts[d].size(); ++k) {
            const int s = parts[d][k];
            out->shards[s] = sub_shards[d][k];
            out->shards[s].valid = merged[s];
            if (device_of_shard) device_of_shard[s] = d;
        }
        if (!parts[d].empty()) {
            out->n_suspect += sub_out[d].n_suspect;
            out->raia_valid = std::max(out->raia_valid, sub_out[d].raia_valid);
            out->seconds_kernel = std::max(out->seconds_kernel, sub_out[d].seconds_kernel);
        }
    }
    for (int s = 0; s < ns; ++s) {
        out->valid = std::max(out->valid, out->shards[s].valid);
        out->n_failures += out->shards[s].valid != JTB_VALID;
    }
    out->seconds_total = now_s() - t0;
    return 0;
}

}  // extern "C"
