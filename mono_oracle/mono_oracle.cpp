// mono_oracle.cpp — CPU oracle of the monotonic-key check (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// MONO_GRAPH restates src/tigerbeetle/elle/core.clj literally: for every key the :ok reads are grouped by the value
// they observed, the groups are sorted by value and consecutive groups are linked.  Linking every read of group i to
// every read of group i+1 is quadratic, so one virtual node per consecutive pair stands between them
// (group_i -> virt_i -> group_i+1): read r reaches read s through the virtual nodes of key k iff v_k(r) < v_k(s),
// which is the transitive closure of monotonic-key-order and so has the same cycles.  Real-time edges go through a
// chain of virtual nodes T_0 -> T_1 -> ... over the event positions of the shard: r -> T_comp(r), T_(inv(s)-1) -> s,
// so r reaches s iff r completed before s was invoked.  Virtual nodes only ever lie on paths between reads, so the
// graph has a cycle iff the read graph does; an iterative Tarjan SCC search decides it.  It is exact on shards with
// partial reads too (MONO_DECIDE_PARTIAL).
// MONO_PAIRS decides "there is a 2-cycle" by brute force over all pairs of reads (O(n^2), small histories only).
// Both report the witness through a binary search over the completion-position prefix and the partner through a
// brute-force scan of the witness' prefix.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../include/jtb_check.h"

namespace {

constexpr int MONO_GRAPH = 0, MONO_PAIRS = 1;
constexpr int32_t MONO_DECIDE_PARTIAL = 1 << 16;   // oracle only: decide shards with partial reads instead of UNKNOWN

thread_local std::string g_err;

struct Read {
    int32_t inv, comp, comp_index, inv_index;
    std::vector<std::pair<int32_t, int64_t>> kv;   // sorted by key
};

// v(x) < v(y) on some key both read: the smallest such key, or INT64_MIN sentinel via found=false
bool mono_edge(const Read& x, const Read& y, int32_t* key, int64_t* vx, int64_t* vy) {
    size_t i = 0, j = 0;
    while (i < x.kv.size() && j < y.kv.size()) {
        if (x.kv[i].first < y.kv[j].first) ++i;
        else if (x.kv[i].first > y.kv[j].first) ++j;
        else {
            if (x.kv[i].second < y.kv[j].second) {
                if (key) { *key = x.kv[i].first; *vx = x.kv[i].second; *vy = y.kv[j].second; }
                return true;
            }
            ++i, ++j;
        }
    }
    return false;
}

bool edge(const Read& x, const Read& y, bool rt) { return mono_edge(x, y, nullptr, nullptr, nullptr) || (rt && x.comp < y.inv); }

// iterative Tarjan: is there an SCC with more than one node?
bool has_cycle(int n, const std::vector<int64_t>& off, const std::vector<int32_t>& adj) {
    std::vector<int32_t> idx(n, -1), low(n, 0), stack;
    std::vector<char> on(n, 0);
    std::vector<std::pair<int32_t, int64_t>> call;   // (node, next edge)
    int32_t counter = 0;
    for (int32_t root = 0; root < n; ++root) {
        if (idx[root] >= 0) continue;
        call.push_back({root, off[root]});
        idx[root] = low[root] = counter++;
        stack.push_back(root);
        on[root] = 1;
        while (!call.empty()) {
            auto& [v, e] = call.back();
            if (e < off[v + 1]) {
                const int32_t w = adj[e++];
                if (idx[w] < 0) {
                    idx[w] = low[w] = counter++;
                    stack.push_back(w);
                    on[w] = 1;
                    call.push_back({w, off[w]});
                } else if (on[w]) low[v] = std::min(low[v], idx[w]);
                continue;
            }
            const int32_t vv = v;
            call.pop_back();
            if (!call.empty()) low[call.back().first] = std::min(low[call.back().first], low[vv]);
            if (low[vv] == idx[vv]) {
                int size = 0;
                int32_t w;
                do {
                    w = stack.back();
                    stack.pop_back();
                    on[w] = 0;
                    ++size;
                } while (w != vv);
                if (size > 1) return true;
            }
        }
    }
    return false;
}

// the literal graph over the reads with comp <= bound
bool graph_cyclic(const std::vector<Read>& R, int32_t n_pos, int32_t bound, bool rt) {
    std::vector<int32_t> sel;
    for (int32_t i = 0; i < (int32_t)R.size(); ++i)
        if (R[i].comp <= bound) sel.push_back(i);
    const int32_t n = (int32_t)sel.size();
    std::vector<std::pair<int32_t, int32_t>> E;
    int32_t next = n;
    // monotonic: per key, the reads grouped by value in ascending value order; consecutive groups linked
    struct KV { int32_t key; int64_t value; int32_t read; };
    std::vector<KV> obs;
    for (int32_t i = 0; i < n; ++i)
        for (auto& [k, v] : R[sel[i]].kv) obs.push_back({k, v, i});
    std::sort(obs.begin(), obs.end(), [](const KV& x, const KV& y) {
        return x.key != y.key ? x.key < y.key : x.value != y.value ? x.value < y.value : x.read < y.read;
    });
    for (size_t g = 0; g < obs.size();) {   // g: first observation of a (key, value) group
        size_t e = g;
        while (e < obs.size() && obs[e].key == obs[g].key && obs[e].value == obs[g].value) ++e;
        if (e < obs.size() && obs[e].key == obs[g].key) {   // the next group of the same key
            size_t f = e;
            while (f < obs.size() && obs[f].key == obs[e].key && obs[f].value == obs[e].value) ++f;
            const int32_t virt = next++;
            for (size_t a = g; a < e; ++a) E.push_back({obs[a].read, virt});
            for (size_t b = e; b < f; ++b) E.push_back({virt, obs[b].read});
        }
        g = e;
    }
    if (rt && n_pos > 0) {
        const int32_t T0 = next;
        next += n_pos;
        for (int32_t p = 0; p + 1 < n_pos; ++p) E.push_back({T0 + p, T0 + p + 1});
        for (int32_t i = 0; i < n; ++i) {
            const Read& r = R[sel[i]];
            E.push_back({i, T0 + r.comp});
            if (r.inv >= 1) E.push_back({T0 + r.inv - 1, i});
        }
    }
    std::vector<int64_t> off(next + 1, 0);
    for (auto& e : E) off[e.first + 1]++;
    for (int32_t v = 0; v < next; ++v) off[v + 1] += off[v];
    std::vector<int32_t> adj(E.size());
    std::vector<int64_t> fill(off.begin(), off.end() - 1);
    for (auto& e : E) adj[fill[e.first]++] = e.second;
    return has_cycle(next, off, adj);
}

bool pairs_cyclic(const std::vector<Read>& R, int32_t bound, bool rt) {
    for (size_t i = 0; i < R.size(); ++i) {
        if (R[i].comp > bound) continue;
        for (size_t j = i + 1; j < R.size(); ++j)
            if (R[j].comp <= bound && edge(R[i], R[j], rt) && edge(R[j], R[i], rt)) return true;
    }
    return false;
}

void explain(const Read& x, const Read& y, bool rt, jtb_mono_shard& o, int slot) {
    int32_t key;
    int64_t vx, vy;
    o.edge_kind[slot] = JTB_MONO_EDGE_NONE;
    o.edge_key[slot] = -1;
    o.edge_value[slot] = o.edge_value2[slot] = 0;
    if (mono_edge(x, y, &key, &vx, &vy)) {
        o.edge_kind[slot] = JTB_MONO_EDGE_MONOTONIC;
        o.edge_key[slot] = key;
        o.edge_value[slot] = vx;
        o.edge_value2[slot] = vy;
    } else if (rt && x.comp < y.inv) {
        o.edge_kind[slot] = JTB_MONO_EDGE_REALTIME;
        o.edge_value[slot] = x.comp_index;
        o.edge_value2[slot] = y.inv_index;
    }
}

}  // namespace

extern "C" {

const char* jtbm_last_error(void) { return g_err.c_str(); }

int jtbm_check_monotonic_keys(const jtb_history* h, int32_t flags, int32_t algo, jtb_mono_shard* shards,
                              jtb_mono_result* out) {
    const auto t0 = std::chrono::steady_clock::now();
    const bool rt = !(flags & JTB_MONO_NO_REALTIME), decide_partial = flags & MONO_DECIDE_PARTIAL;
    memset(out, 0, sizeof *out);
    char buf[256];
    int64_t total_reads = 0;
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
        std::unordered_map<int32_t, std::pair<int32_t, int32_t>> last_inv;   // process -> (position, :index)
        std::vector<Read> R;
        std::map<int32_t, int> keys;
        for (int64_t e = lo; e < hi; ++e) {
            const int32_t p = h->process[e];
            if (p < 0) continue;
            if (h->type[e] == JTB_T_INVOKE) { last_inv[p] = {(int32_t)(e - lo), h->index[e]}; continue; }
            if (h->type[e] != JTB_T_OK || h->f[e] != JTB_F_READ || h->payload_len[e] < 0) continue;
            const int32_t len = h->payload_len[e];
            const int64_t off = h->payload_off[e];
            if (len % 3 != 0 || off < 0 || off + len > h->n_payload) {
                snprintf(buf, sizeof buf, "read at :index %d: malformed payload", h->index[e]);
                g_err = buf;
                return -2;
            }
            Read r;
            auto it = last_inv.find(p);
            r.inv = it == last_inv.end() ? -1 : it->second.first;
            r.inv_index = it == last_inv.end() ? -1 : it->second.second;
            r.comp = (int32_t)(e - lo);
            r.comp_index = h->index[e];
            for (int32_t j = 0; j < len; j += 3) {
                const int32_t* t = h->payload + off + j;
                r.kv.push_back({t[0], (int64_t)(((uint64_t)(uint32_t)t[2] << 32) | (uint32_t)t[1])});
                keys[t[0]] = 1;
            }
            std::sort(r.kv.begin(), r.kv.end());
            for (size_t j = 1; j < r.kv.size(); ++j)
                if (r.kv[j].first == r.kv[j - 1].first) {
                    snprintf(buf, sizeof buf, "read at :index %d observes key %d twice", h->index[e], r.kv[j].first);
                    g_err = buf;
                    return -2;
                }
            R.push_back(std::move(r));
        }
        total_reads += (int64_t)R.size();
        jtb_mono_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.n_reads = (int32_t)R.size();
        o.n_keys = (int32_t)keys.size();
        o.witness_index = o.partner_index = -1;
        o.edge_key[0] = o.edge_key[1] = -1;
        bool partial = false;
        for (auto& r : R) partial |= r.kv.size() < keys.size();
        if (partial && !decide_partial) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_PARTIAL_READ;
            continue;
        }
        const int32_t n_pos = (int32_t)(hi - lo);
        auto cyclic = [&](int32_t bound) {
            return algo == MONO_PAIRS ? pairs_cyclic(R, bound, rt) : graph_cyclic(R, n_pos, bound, rt);
        };
        if (R.size() < 2 || !cyclic(INT_MAX)) continue;
        o.valid = JTB_INVALID;
        int32_t a = 0, b = n_pos - 1;
        while (a < b) {
            const int32_t mid = (a + b) / 2;
            if (cyclic(mid)) b = mid; else a = mid + 1;
        }
        o.witness_index = h->index[lo + b];
        const Read* w = nullptr;
        for (auto& r : R)
            if (r.comp == b) w = &r;
        const Read* partner = nullptr;
        for (auto& r : R)
            if (&r != w && r.comp <= b && edge(r, *w, rt) && edge(*w, r, rt) &&
                (!partner || r.comp_index < partner->comp_index))
                partner = &r;
        if (partner) {
            o.partner_index = partner->comp_index;
            explain(*partner, *w, rt, o, 0);
            explain(*w, *partner, rt, o, 1);
        }
    }
    out->n_reads = total_reads;
    for (int32_t s = 0; s < h->n_shards; ++s) {
        out->valid = std::max(out->valid, shards[s].valid);
        if (shards[s].valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
