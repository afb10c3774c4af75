// counter_bounds.cpp — CPU oracle of the counter-bounds check (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// Both deciders parse a shard the same plain way (reads paired with the latest invoke of their process, transfers with
// the next event of their process) and fill jtb_cb_shard exactly as jtb_check_counter_bounds does.
// CB_LITERAL restates the definition: for every (read, key) it sums over every transfer of the shard, O(R * K * T).
// CB_SWEEP walks the events once keeping running sums per key: U grows at every non-:fail transfer invocation, L at
// every :ok transfer completion; a read snapshots L at its invocation and compares at its completion.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../include/jtb_check.h"

namespace {

constexpr int CB_LITERAL = 0, CB_SWEEP = 1;

thread_local std::string g_err;

struct CRead {
    int32_t inv, comp, comp_index;
    std::vector<std::pair<int32_t, int64_t>> kv;   // sorted by key
};

struct CTransfer {
    int32_t inv, comp, inv_index, comp_index;   // comp = position of the fate event, -1 = never completed
    int32_t fate;                               // JTB_T_OK / _INFO / _FAIL, -1 = none
    int32_t amount, debit, credit;
    bool touches(int32_t k) const { return k == 2 * debit || k == 2 * credit + 1; }
};

int parse_shard(const jtb_history* h, int32_t s, std::vector<CRead>& R, std::vector<CTransfer>& T) {
    const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
    std::unordered_map<int32_t, int32_t> last_inv;   // process -> position of its latest invoke
    std::unordered_map<int32_t, size_t> open;        // process -> its transfer awaiting a fate
    char buf[256];
    for (int64_t e = lo; e < hi; ++e) {
        const int32_t p = h->process[e], pos = (int32_t)(e - lo);
        if (p < 0) continue;
        auto ot = open.find(p);
        if (ot != open.end()) {
            if (h->type[e] != JTB_T_INVOKE) {
                T[ot->second].fate = h->type[e];
                T[ot->second].comp = pos;
                T[ot->second].comp_index = h->index[e];
            }
            open.erase(ot);
        }
        if (h->type[e] == JTB_T_INVOKE) {
            last_inv[p] = pos;
            if (h->f[e] == JTB_F_TRANSFER) {
                if (h->a[e] < 0) {
                    snprintf(buf, sizeof buf, "transfer at :index %d: negative amount %d", h->index[e], h->a[e]);
                    g_err = buf;
                    return -2;
                }
                if (h->b[e] < 0 || h->b[e] >= (1 << 30) || h->c[e] < 0 || h->c[e] >= (1 << 30)) {
                    snprintf(buf, sizeof buf, "transfer at :index %d: account outside [0, 2^30)", h->index[e]);
                    g_err = buf;
                    return -2;
                }
                open[p] = T.size();
                T.push_back({pos, -1, h->index[e], -1, -1, h->a[e], h->b[e], h->c[e]});
            }
            continue;
        }
        if (h->type[e] != JTB_T_OK || h->f[e] != JTB_F_READ || h->payload_len[e] < 0) continue;
        const int32_t len = h->payload_len[e];
        const int64_t off = h->payload_off[e];
        if (len % 3 != 0 || off < 0 || off + len > h->n_payload) {
            snprintf(buf, sizeof buf, "read at :index %d: malformed payload", h->index[e]);
            g_err = buf;
            return -2;
        }
        CRead r;
        auto it = last_inv.find(p);
        r.inv = it == last_inv.end() ? -1 : it->second;
        r.comp = pos;
        r.comp_index = h->index[e];
        for (int32_t j = 0; j < len; j += 3) {
            const int32_t* t = h->payload + off + j;
            r.kv.push_back({t[0], (int64_t)(((uint64_t)(uint32_t)t[2] << 32) | (uint32_t)t[1])});
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
    return 0;
}

bool in_L(const CTransfer& t, const CRead& r) { return t.fate == JTB_T_OK && r.inv >= 0 && t.comp < r.inv; }
bool in_U(const CTransfer& t, const CRead& r) { return t.fate != JTB_T_FAIL && t.inv < r.comp; }

// the culprit of a BELOW witness: the first transfer of L, in completion order, at which the running sum exceeds v
int32_t below_culprit(const std::vector<CTransfer>& T, const CRead& r, int32_t k, int64_t v) {
    std::vector<const CTransfer*> in;
    for (auto& t : T)
        if (t.touches(k) && in_L(t, r)) in.push_back(&t);
    std::sort(in.begin(), in.end(), [](const CTransfer* x, const CTransfer* y) { return x->comp < y->comp; });
    int64_t run = 0;
    for (auto* t : in)
        if ((run += t->amount) > v) return t->comp_index;
    return -1;
}

void decide_literal(const std::vector<CRead>& R, const std::vector<CTransfer>& T, jtb_cb_shard& o) {
    for (auto& r : R)
        for (auto& [k, v] : r.kv) {
            int64_t L = 0, U = 0;
            const CTransfer* last = nullptr;   // the transfer of U invoked last
            for (auto& t : T) {
                if (!t.touches(k)) continue;
                if (in_L(t, r)) L += t.amount;
                if (in_U(t, r)) {
                    U += t.amount;
                    if (!last || t.inv > last->inv) last = &t;
                }
            }
            if (v >= L && v <= U) continue;
            (v < L ? o.n_below : o.n_above)++;
            if (o.valid == JTB_INVALID) continue;   // reads and keys are visited in witness order: the first one wins
            o.valid = JTB_INVALID;
            o.witness_index = r.comp_index;
            o.witness_key = k;
            o.value = v;
            o.kind = v < L ? JTB_CB_BELOW : JTB_CB_ABOVE;
            o.bound = v < L ? L : U;
            o.culprit_index = v < L ? below_culprit(T, r, k, v) : (last ? last->inv_index : -1);
        }
}

void decide_sweep(int32_t n_pos, const std::vector<CRead>& R, const std::vector<CTransfer>& T, jtb_cb_shard& o) {
    std::unordered_map<int32_t, int32_t> kid;   // observed key -> dense id
    for (auto& r : R)
        for (auto& kv : r.kv) kid.emplace(kv.first, (int32_t)kid.size());
    // what happens at each position: a transfer's invocation or :ok completion, a read's invocation or completion
    std::vector<int32_t> t_inv(n_pos, -1), t_ok(n_pos, -1), r_comp(n_pos, -1);
    std::vector<std::vector<int32_t>> r_inv(n_pos);
    for (int32_t i = 0; i < (int32_t)T.size(); ++i) {
        if (T[i].fate != JTB_T_FAIL) t_inv[T[i].inv] = i;
        if (T[i].fate == JTB_T_OK) t_ok[T[i].comp] = i;
    }
    for (int32_t i = 0; i < (int32_t)R.size(); ++i) {
        r_comp[R[i].comp] = i;
        if (R[i].inv >= 0) r_inv[R[i].inv].push_back(i);
    }
    const size_t nk = kid.size();
    std::vector<int64_t> sumL(nk, 0), sumU(nk, 0);
    std::vector<int32_t> lastU(nk, -1);   // invocation :index of the last transfer counted in U
    std::vector<std::vector<int64_t>> snapL(R.size());
    auto add = [&](const CTransfer& t, std::vector<int64_t>& sum, bool mark) {
        const int32_t ks[2] = {2 * t.debit, 2 * t.credit + 1};
        for (int32_t k : ks) {
            auto it = kid.find(k);
            if (it == kid.end()) continue;
            sum[it->second] += t.amount;
            if (mark) lastU[it->second] = t.inv_index;
        }
    };
    for (int32_t pos = 0; pos < n_pos; ++pos) {
        if (t_inv[pos] >= 0) add(T[t_inv[pos]], sumU, true);
        if (t_ok[pos] >= 0) add(T[t_ok[pos]], sumL, false);
        for (int32_t i : r_inv[pos]) {
            snapL[i].resize(R[i].kv.size());
            for (size_t j = 0; j < R[i].kv.size(); ++j) snapL[i][j] = sumL[kid[R[i].kv[j].first]];
        }
        if (r_comp[pos] < 0) continue;
        const CRead& r = R[r_comp[pos]];
        const auto& snap = snapL[r_comp[pos]];
        for (size_t j = 0; j < r.kv.size(); ++j) {
            const int32_t k = r.kv[j].first, id = kid[k];
            const int64_t v = r.kv[j].second, L = snap.empty() ? 0 : snap[j], U = sumU[id];
            if (v >= L && v <= U) continue;
            (v < L ? o.n_below : o.n_above)++;
            if (o.valid == JTB_INVALID) continue;
            o.valid = JTB_INVALID;
            o.witness_index = r.comp_index;
            o.witness_key = k;
            o.value = v;
            o.kind = v < L ? JTB_CB_BELOW : JTB_CB_ABOVE;
            o.bound = v < L ? L : U;
            if (v > U) {
                o.culprit_index = lastU[id];
            } else {   // a second walk over the :ok completions before the read's invocation
                int64_t run = 0;
                for (int32_t q = 0; q < r.inv; ++q)
                    if (t_ok[q] >= 0 && T[t_ok[q]].touches(k) && (run += T[t_ok[q]].amount) > v) {
                        o.culprit_index = T[t_ok[q]].comp_index;
                        break;
                    }
            }
        }
    }
}

}  // namespace

extern "C" {

const char* jtbm_cb_last_error(void) { return g_err.c_str(); }

int jtbm_check_counter_bounds(const jtb_history* h, int32_t flags, int32_t algo, jtb_cb_shard* shards,
                              jtb_cb_result* out) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    memset(out, 0, sizeof *out);
    for (int32_t s = 0; s < h->n_shards; ++s) {
        std::vector<CRead> R;
        std::vector<CTransfer> T;
        if (int rc = parse_shard(h, s, R, T)) return rc;
        jtb_cb_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        o.n_reads = (int32_t)R.size();
        std::vector<int32_t> keys;
        for (auto& r : R)
            for (auto& kv : r.kv) keys.push_back(kv.first);
        std::sort(keys.begin(), keys.end());
        o.n_keys = (int32_t)(std::unique(keys.begin(), keys.end()) - keys.begin());
        for (auto& t : T) o.n_transfers += t.fate != JTB_T_FAIL;
        o.witness_index = o.witness_key = o.culprit_index = -1;
        if (algo == CB_SWEEP) decide_sweep((int32_t)(h->shard_off[s + 1] - h->shard_off[s]), R, T, o);
        else decide_literal(R, T, o);
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_violations += o.n_below + o.n_above;
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
