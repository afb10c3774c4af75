// read_gaps.cpp — CPU oracle of the read-gap check (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// Both deciders parse a shard the way the read-explanation oracle does (reads and lookups paired with the latest invoke
// of their process, every [:t ...] micro-op a transfer paired with the next event of its process, M(t) and A(t) from
// the lookups), order the :ok reads of a full-key shard by (S as 128 bits, invocation position), stably over completion
// order, and decide every gap between successive reads; they fill jtb_rg_shard as jtb_check_read_gaps does.
// RG_BRUTE is the definition: every subset of a gap's eligible transfers that fit under Delta (no member of a solution
// exceeds Delta_k on a key; the kinds are defined over these), no caps (tiny histories only); a transfer in every
// solution of two gaps is DOUBLE.
// RG_SEARCH is the library's decision: the amount filter while gathering, the same caps, the root pruning fixpoint in
// Jacobi rounds, at most 64 free candidates in the canonical order (amount descending, then id), a depth-first search
// including before excluding, the same fixpoint at every node and the node budget; a transfer the root pruning forces
// into two gaps is DOUBLE.  Node counts are the library's.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../include/jtb_check.h"

#include "gaps_common.h"

namespace {

// one gap: upper read u, lower read l (nullptr for gap 0); X: RG_SEARCH's sweep (nullptr: RG_BRUTE)
GapOut decide_gap(const Shard& S, const std::vector<int32_t>& keys, const Index* X, const XRead& u, const XRead* l,
                  int algo, int64_t max_nodes, int64_t& nodes) {
    GapOut o;
    const int32_t K = (int32_t)keys.size();
    if (algo == RG_SEARCH && K > JTB_RG_MAX_KEYS) { o.code = G_UNDECIDED; return o; }
    Problem pb;
    pb.key = keys;
    pb.d.resize(K);
    bool nz = false;
    for (int32_t j = 0; j < K; ++j) {
        pb.d[j] = u.kv[j].second - (l ? l->kv[j].second : 0);
        if (pb.d[j] < 0) { o.code = JTB_RG_KEY; o.key = keys[j]; o.delta = pb.d[j]; return o; }
        nz |= pb.d[j] != 0;
    }
    if (!nz) return o;
    const int32_t ivl = l ? l->inv : -1;
    auto take = [&](int32_t t) {   // false: more eligible transfers than the gather cap
        const XTransfer& x = S.T[t];
        if (x.fate == JTB_T_FAIL || !(x.inv < u.comp) || !(x.A < u.comp) || x.M < ivl || x.amount <= 0) return true;
        const int32_t jd = col_of(keys, 2 * (int64_t)x.debit), jc = col_of(keys, 2 * (int64_t)x.credit + 1);
        if (jd < 0 && jc < 0) return true;
        if ((jd >= 0 && x.amount > pb.d[jd]) || (jc >= 0 && x.amount > pb.d[jc])) return true;   // fits under Delta
        pb.P.push_back({x.id, x.amount, jd, jc, t});
        return !X || pb.P.size() <= (size_t)JTB_RG_MAX_GATHER;
    };
    bool fits = true;
    if (!X) {
        for (int32_t t = 0; t < (int32_t)S.T.size(); ++t) take(t);
    } else {
        // :ok transfers invoked before u completed, back to the last one whose running max completion is before l's
        // invocation (every earlier one completed before it, so is in l's state); the crashed ones anchored at a key
        // that grew
        for (int64_t j = std::lower_bound(X->ok_inv.begin(), X->ok_inv.end(), u.comp) - X->ok_inv.begin() - 1;
             fits && j >= 0 && X->ok_pmax[j] >= ivl; --j)
            fits = take(X->ok[j]);
        for (int32_t c = 0; c < K && fits; ++c) {
            if (pb.d[c] <= 0) continue;
            const int64_t bc = std::lower_bound(X->crashed_inv[c].begin(), X->crashed_inv[c].end(), u.comp) -
                               X->crashed_inv[c].begin();
            for (int64_t j = 0; j < bc && fits; ++j) fits = take(X->crashed[c][j]);
        }
    }
    if (algo == RG_BRUTE) {
        o.n_eligible = (int32_t)pb.P.size();
        uint64_t all;
        if (brute(pb, -1, false, all)) {
            for (size_t c = 0; c < pb.P.size(); ++c)
                if (all >> c & 1) o.forced.push_back(pb.P[c].t);
            return o;
        }
        o.code = JTB_RG_JOINT;
        for (int32_t k = 0; k < K; ++k)
            if (!brute(pb, k, true, all)) { o.code = JTB_RG_KEY; o.key = keys[k]; o.delta = pb.d[k]; break; }
        return o;
    }
    if (!fits) { o.code = G_UNDECIDED; return o; }
    Search s(pb, -1, max_nodes);
    int32_t root_key, kept;
    std::vector<int32_t> forced;
    const Verdict v = s.run(root_key, kept, &forced);
    nodes += s.nodes;
    o.n_eligible = kept;
    for (int32_t c : forced) o.forced.push_back(pb.P[c].t);
    if (v == EXPLAINED) return o;
    if (v == UNDECIDED) { o.code = G_UNDECIDED; return o; }
    o.code = JTB_RG_JOINT;
    o.key = root_key;
    for (int32_t k = 0; k < K; ++k) {
        Search sk(pb, k, max_nodes);
        int32_t rk, kp;
        const Verdict vk = sk.run(rk, kp);
        nodes += sk.nodes;
        if (vk == UNEXPLAINED) { o.code = JTB_RG_KEY; o.key = keys[k]; o.delta = pb.d[k]; break; }
    }
    return o;
}

}  // namespace

extern "C" {

const char* jtbm_rg_last_error(void) { return g_err.c_str(); }

// per_gap (may be NULL): one code per :ok read in shard-major order, the gaps of a full-key shard in gap order, 3 for
// the reads of a partial-read shard: 0 explained, 1 KEY, 2 JOINT, 3 undecided
int jtbm_check_read_gaps(const jtb_history* h, int64_t max_nodes, int32_t flags, int32_t algo, jtb_rg_shard* shards,
                         jtb_rg_result* out, int8_t* per_gap) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (max_nodes <= 0) max_nodes = JTB_RG_DEFAULT_MAX_NODES;
    memset(out, 0, sizeof *out);
    int64_t n_records = 0, n_reads = 0;
    std::vector<jtb_rg_shard> tmp(h->n_shards);
    std::vector<int8_t> codes;
    try {
        for (int32_t s = 0; s < h->n_shards; ++s) {
            Shard S;
            if (int rc = parse_shard(h, s, S, n_records)) return rc;
            n_reads += (int64_t)S.R.size();
            if (n_reads > INT_MAX) { g_err = "more than 2^31-1 reads"; return -2; }
            classify_inputs(S);
            jtb_rg_shard& o = tmp[s];
            memset(&o, 0, sizeof o);
            o.valid = JTB_VALID;
            o.n_reads = (int32_t)S.R.size();
            o.n_transfers = (int32_t)S.T.size();
            o.witness_index = o.lower_index = o.key = o.other_index = -1;
            std::vector<int32_t> keys;
            for (auto& r : S.R)
                for (auto& kv : r.kv) keys.push_back(kv.first);
            std::sort(keys.begin(), keys.end());
            keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
            bool partial = false;
            for (auto& r : S.R) partial |= r.kv.size() < keys.size();
            if (partial) {
                o.valid = JTB_UNKNOWN;
                o.cause = JTB_CAUSE_PARTIAL_READ;
                codes.insert(codes.end(), S.R.size(), G_UNDECIDED);
                continue;
            }
            // the gap order: (S, invocation), stable over completion order
            std::vector<int32_t> ord(S.R.size());
            std::vector<__int128> sum(S.R.size(), 0);
            for (size_t r = 0; r < S.R.size(); ++r) {
                ord[r] = (int32_t)r;
                for (auto& kv : S.R[r].kv) sum[r] += kv.second;
            }
            std::stable_sort(ord.begin(), ord.end(), [&](int32_t a, int32_t b) {
                return sum[a] != sum[b] ? sum[a] < sum[b] : S.R[a].inv < S.R[b].inv;
            });
            const int32_t n = (int32_t)ord.size();
            std::vector<GapOut> g(n);
            std::map<int32_t, std::vector<int32_t>> forced_in;   // transfer -> gaps forcing it in, ascending
            std::unique_ptr<Index> X;
            if (algo == RG_SEARCH) X.reset(new Index(S, keys));
            for (int32_t i = 0; i < n; ++i) {
                g[i] = decide_gap(S, keys, X.get(), S.R[ord[i]], i > 0 ? &S.R[ord[i - 1]] : nullptr, algo, max_nodes,
                                  o.nodes);
                codes.push_back(g[i].code);
                if (g[i].code == G_EXPLAINED) o.n_explained++;
                else if (g[i].code == G_UNDECIDED) o.n_undecided++;
                else o.count_by_kind[g[i].code - 1]++;
                for (int32_t t : g[i].forced) forced_in[t].push_back(i);
            }
            // the witness: the first violating gap, the smallest kind there, the smallest DOUBLE id there
            int32_t wgap = INT_MAX, wkind = 0, wt = -1;
            for (int32_t i = 0; i < n && wgap == INT_MAX; ++i)
                if (g[i].code == JTB_RG_KEY || g[i].code == JTB_RG_JOINT) { wgap = i; wkind = g[i].code; }
            for (auto& [t, gs] : forced_in) {
                if (gs.size() < 2) continue;
                o.count_by_kind[2]++;
                if (gs[1] < wgap || (gs[1] == wgap && wkind == JTB_RG_DOUBLE && S.T[t].id < S.T[wt].id)) {
                    wgap = gs[1];
                    wkind = JTB_RG_DOUBLE;
                    wt = t;
                }
            }
            if (wgap == INT_MAX) {
                o.valid = o.n_undecided ? JTB_UNKNOWN : JTB_VALID;
                continue;
            }
            o.valid = JTB_INVALID;
            o.kind = wkind;
            o.witness_index = S.R[ord[wgap]].comp_index;
            o.lower_index = wgap > 0 ? S.R[ord[wgap - 1]].comp_index : -1;
            o.n_eligible = g[wgap].n_eligible;
            if (wkind == JTB_RG_DOUBLE) {
                o.transfer_id = S.T[wt].id;
                o.other_index = S.R[ord[forced_in[wt][0]]].comp_index;
            } else {
                o.key = g[wgap].key;
                o.delta = g[wgap].delta;
            }
        }
    } catch (int) {
        return -2;
    }
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const jtb_rg_shard& o = shards[s] = tmp[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_explained += o.n_explained;
        out->n_unexplained += o.count_by_kind[0] + o.count_by_kind[1];
        out->n_double += o.count_by_kind[2];
        out->n_undecided += o.n_undecided;
        out->nodes += o.nodes;
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    if (per_gap) std::copy(codes.begin(), codes.end(), per_gap);
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
