// lookup_witness.cpp — CPU oracles of the lookup witness (TEST INFRASTRUCTURE ONLY; the library never calls them).
//
// LK_SEARCH is the library's decision, shard by shard: CW_SEARCH, then on every shard it proves that has an :ok lookup
// the placement of the lookups in its serial order (DESIGN.md "K17 lookup witness"): the commit gaps G(t) from
// CW_SEARCH's commit_read, every lookup's allowed range [lo, hi] and its position, the nesting of the lookups of one gap,
// and one greedy real-time pass over the merged order of reads, transfers and lookups.
//
// LK_BRUTE is the definition on tiny histories: whether some serial order of the reads, the :ok transfers, any subset
// of the crashed transfers and the :ok lookups respects real time, gives every read its counters and every lookup
// exactly the transfers committed before it.  valid is JTB_VALID when one exists, else JTB_INVALID.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <unordered_map>
#include <unordered_set>

#include "gaps_common.h"

extern "C" int jtbm_check_class_witness(const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                                        int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t algo,
                                        int32_t* commit_read, jtb_cw_shard* shards, jtb_cw_result* out);
extern "C" const char* jtbm_cw_last_error(void);

namespace {

constexpr int LK_BRUTE = 0, LK_SEARCH = 1;
constexpr int32_t NEVER = INT_MAX;   // G(t) of a transfer that never commits

struct LRec {
    int64_t id;
    int32_t debit, credit, amount;
};
struct LLookup {
    int32_t inv, comp, comp_index;
    std::vector<LRec> rec;
};

// the :ok lookups of shard s with their records, in completion order (parse_shard pairs them the same way)
std::vector<LLookup> parse_lookups(const jtb_history* h, int32_t s) {
    std::vector<LLookup> L;
    std::unordered_map<int32_t, int32_t> last_inv;
    const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
    for (int64_t e = lo; e < hi; ++e) {
        const int32_t p = h->process[e], pos = (int32_t)(e - lo);
        if (p < 0) continue;
        if (h->type[e] == JTB_T_INVOKE) {
            last_inv[p] = pos;
            continue;
        }
        if (h->type[e] != JTB_T_OK || h->f[e] != JTB_F_LOOKUP || h->payload_len[e] < 0) continue;
        auto it = last_inv.find(p);
        LLookup l{it == last_inv.end() ? -1 : it->second, pos, h->index[e], {}};
        const int32_t* r = h->payload + h->payload_off[e];
        for (int32_t j = 0; j < h->payload_len[e]; j += 5) l.rec.push_back({rec_id(r + j), r[j + 2], r[j + 3], r[j + 4]});
        L.push_back(std::move(l));
    }
    return L;
}

// the lookup pass on one shard CW_SEARCH proves; o, commit (the shard's transfers) and lread (its :ok lookups) are
// updated in place
void lookup_pass(const Shard& S, const std::vector<int32_t>& ord, const std::vector<LLookup>& L, jtb_lk_shard& o,
                 std::vector<int32_t>& commit, std::vector<int32_t>& lread) {
    const int32_t n = (int32_t)ord.size(), nT = (int32_t)S.T.size(), nL = (int32_t)L.size();
    std::unordered_map<int32_t, int32_t> pos_of;   // completion :index of a read -> its position
    for (int32_t i = 0; i < n; ++i) pos_of[S.R[ord[i]].comp_index] = i;
    std::unordered_map<int64_t, int32_t> tix;
    for (int32_t t = 0; t < nT; ++t) tix[S.T[t].id] = t;
    std::vector<char> shown(nT, 0);
    for (const LLookup& l : L)
        for (const LRec& r : l.rec) {
            auto it = tix.find(r.id);
            if (it != tix.end()) shown[it->second] = 1;
        }
    // the commit gaps
    std::vector<int32_t> G(nT, NEVER);
    for (int32_t t = 0; t < nT; ++t) {
        const XTransfer& z = S.T[t];
        if (commit[t] >= 0) G[t] = pos_of.at(commit[t]);
        else if (z.fate == JTB_T_OK || (z.fate != JTB_T_FAIL && shown[t])) G[t] = n;
    }
    // N[g] = committed transfers with G <= g, g in [0, n]
    std::vector<int64_t> N(n + 1, 0);
    for (int32_t t = 0; t < nT; ++t)
        if (G[t] != NEVER) N[G[t]]++;
    for (int32_t g = 1; g <= n; ++g) N[g] += N[g - 1];
    auto nlt = [&](int32_t g) { return g > 0 ? N[g - 1] : 0; };
    // K13's points of the reads: Q[i] = max(Q[i-1], iv(r_i), iv(t) for t in D_i)
    std::vector<int32_t> gmax(n, INT_MIN), Q(n);
    for (int32_t t = 0; t < nT; ++t)
        if (G[t] < n) gmax[G[t]] = std::max(gmax[G[t]], S.T[t].inv);
    for (int32_t i = 0; i < n; ++i) Q[i] = std::max({i > 0 ? Q[i - 1] : INT_MIN, S.R[ord[i]].inv, gmax[i]});
    auto before = [&](int32_t g) { return g > 0 ? Q[g - 1] : INT_MIN; };   // the point entering gap g
    auto fail = [&](int32_t index) {
        o.valid = JTB_UNKNOWN;
        o.cause = o.lookup_cause = JTB_CAUSE_LOOKUP;
        o.fail_index = o.lookup_fail_index = index;
        o.transfer_id = -1;
        o.n_committed = o.n_committed_crashed = o.n_after = 0;
        std::fill(commit.begin(), commit.end(), JTB_SW_NEVER);
    };
    if (n == 0) return fail(L[0].comp_index);   // a proved shard without reads has no order to place lookups in
    // the allowed ranges and the positions
    std::vector<int32_t> lpos(nL), a(nL);
    for (int32_t l = 0; l < nL; ++l) {
        const LLookup& x = L[l];
        std::unordered_set<int64_t> seen;
        bool bad = false;
        int32_t lo = 0;
        for (const LRec& r : x.rec) {
            auto it = tix.find(r.id);
            if (it == tix.end() || !seen.insert(r.id).second) { bad = true; break; }
            const XTransfer& z = S.T[it->second];
            if (z.debit != r.debit || z.credit != r.credit || z.amount != r.amount || G[it->second] == NEVER) {
                bad = true;
                break;
            }
            lo = std::max(lo, G[it->second]);
        }
        const int64_t k = (int64_t)x.rec.size();
        int64_t slt = 0;
        if (!bad)
            for (const LRec& r : x.rec) slt += G[tix.at(r.id)] < lo;
        if (bad || slt != nlt(lo)) return fail(x.comp_index);
        const int32_t hi = (int32_t)(std::upper_bound(N.begin(), N.end(), k) - N.begin());   // first g: N[g] > k
        int32_t p = lo;
        for (int32_t g = std::min(hi, n); g >= lo; --g)
            if (before(g) < x.comp) { p = g; break; }
        lpos[l] = p;
        a[l] = (int32_t)(k - nlt(p));
    }
    // the lookups of each gap by (position, shown part of D_g, completion); the layers
    std::vector<int32_t> by(nL), rank(nL);
    for (int32_t l = 0; l < nL; ++l) by[l] = l;
    std::sort(by.begin(), by.end(), [&](int32_t u, int32_t v) {
        return lpos[u] != lpos[v] ? lpos[u] < lpos[v] : a[u] != a[v] ? a[u] < a[v] : u < v;
    });
    for (int32_t j = 0; j < nL; ++j) rank[by[j]] = j > 0 && lpos[by[j - 1]] == lpos[by[j]] ? rank[by[j - 1]] + 1 : 0;
    std::vector<int32_t> layer(nT, INT_MAX);
    for (int32_t l = 0; l < nL; ++l)
        for (const LRec& r : L[l].rec) {
            const int32_t t = tix.at(r.id);
            if (G[t] == lpos[l]) layer[t] = std::min(layer[t], rank[l]);
        }
    for (int32_t l = 0; l < nL; ++l) {
        int64_t c = 0;
        for (int32_t t = 0; t < nT; ++t) c += G[t] == lpos[l] && layer[t] <= rank[l];
        if (c != a[l]) return fail(L[l].comp_index);
    }
    // the merged order: (gap, sub, invocation); sub = 2 * layer for a transfer, 2 * rank + 1 for a lookup, then the
    // transfers no lookup of the gap returns, then the read that closes the gap
    struct Op {
        int64_t gp;
        uint32_t sub;
        int32_t iv, cp, kind, i;   // kind 0 read, 1 transfer, 2 lookup
    };
    std::vector<Op> ops;
    for (int32_t i = 0; i < n; ++i) ops.push_back({i, 0xffffffffu, S.R[ord[i]].inv, S.R[ord[i]].comp, 0, i});
    for (int32_t t = 0; t < nT; ++t)
        if (G[t] != NEVER)
            ops.push_back({G[t], layer[t] == INT_MAX ? 0xfffffffeu : 2u * (uint32_t)layer[t], S.T[t].inv,
                           S.T[t].fate == JTB_T_OK ? S.T[t].okcomp : INT_MAX, 1, t});
    for (int32_t l = 0; l < nL; ++l) ops.push_back({lpos[l], 2u * (uint32_t)rank[l] + 1, L[l].inv, L[l].comp, 2, l});
    std::sort(ops.begin(), ops.end(), [](const Op& u, const Op& v) {
        return std::tie(u.gp, u.sub, u.iv) < std::tie(v.gp, v.sub, v.iv);
    });
    int32_t P = INT_MIN, last = -1;
    for (const Op& x : ops) {
        P = std::max(P, x.iv);
        if (x.kind == 2) last = x.i;
        if (P >= x.cp) {
            if (last < 0)   // no lookup precedes the failing op: the shard's first lookup in the merged order
                for (const Op& y : ops)
                    if (y.kind == 2) { last = y.i; break; }
            return fail(L[last].comp_index);
        }
    }
    for (int32_t t = 0; t < nT; ++t)
        if (commit[t] == JTB_SW_NEVER && G[t] == n) commit[t] = JTB_SW_AFTER;
    for (int32_t l = 0; l < nL; ++l) lread[l] = lpos[l] < n ? S.R[ord[lpos[l]]].comp_index : JTB_SW_AFTER;
    o.n_lookups_placed = nL;
}

// ---- LK_BRUTE -------------------------------------------------------------------------------------------------------

// whether shard S with its lookups L has a serial order as the header above states; -1 when it has more than 24 ops
int brute_shard(const Shard& S, const std::vector<LLookup>& L) {
    struct Op {
        int kind, i;   // 0 read, 1 transfer, 2 lookup
        int32_t iv, cp;
        bool required;
    };
    std::vector<Op> ops;
    for (size_t i = 0; i < S.R.size(); ++i) ops.push_back({0, (int)i, S.R[i].inv, S.R[i].comp, true});
    for (size_t t = 0; t < S.T.size(); ++t) {
        const XTransfer& z = S.T[t];
        if (z.fate == JTB_T_FAIL) continue;
        ops.push_back({1, (int)t, z.inv, z.fate == JTB_T_OK ? z.okcomp : INT_MAX, z.fate == JTB_T_OK});
    }
    for (size_t l = 0; l < L.size(); ++l) ops.push_back({2, (int)l, L[l].inv, L[l].comp, true});
    const int n = (int)ops.size();
    if (n > 24) return -1;
    std::unordered_map<int64_t, int32_t> tix;
    for (size_t t = 0; t < S.T.size(); ++t) tix[S.T[t].id] = (int32_t)t;
    auto holds = [&](const Op& x, uint32_t mask) {
        if (x.kind == 1) return true;
        std::vector<char> in(S.T.size(), 0);
        for (int j = 0; j < n; ++j)
            if ((mask >> j & 1) && ops[j].kind == 1) in[ops[j].i] = 1;
        if (x.kind == 0) {
            for (auto& kv : S.R[x.i].kv) {
                int64_t v = 0;
                for (size_t t = 0; t < S.T.size(); ++t)
                    if (in[t]) v += (2 * (int64_t)S.T[t].debit == kv.first ? S.T[t].amount : 0) +
                                    (2 * (int64_t)S.T[t].credit + 1 == kv.first ? S.T[t].amount : 0);
                if (v != kv.second) return false;
            }
            return true;
        }
        std::unordered_set<int64_t> seen;
        size_t shown = 0;
        for (const LRec& r : L[x.i].rec) {
            auto it = tix.find(r.id);
            if (it == tix.end() || !seen.insert(r.id).second || !in[it->second]) return false;
            const XTransfer& z = S.T[it->second];
            if (z.debit != r.debit || z.credit != r.credit || z.amount != r.amount) return false;
            shown++;
        }
        size_t committed = 0;
        for (char c : in) committed += c;
        return shown == committed;
    };
    uint32_t need = 0;
    for (int j = 0; j < n; ++j)
        if (ops[j].required) need |= 1u << j;
    std::unordered_set<uint32_t> seen;
    std::vector<uint32_t> stack{0};
    while (!stack.empty()) {
        const uint32_t mask = stack.back();
        stack.pop_back();
        if ((mask & need) == need) return 1;
        if (!seen.insert(mask).second) continue;
        for (int j = 0; j < n; ++j) {
            if (mask >> j & 1) continue;
            bool ok = true;   // every op left out must not have completed before ops[j] was invoked
            for (int y = 0; y < n && ok; ++y)
                if (y != j && !(mask >> y & 1) && ops[y].cp < ops[j].iv) ok = false;
            if (ok && holds(ops[j], mask)) stack.push_back(mask | 1u << j);
        }
    }
    return 0;
}

}  // namespace

extern "C" {

const char* jtbm_lk_last_error(void) { return g_err.c_str(); }

int jtbm_check_lookup_witness(const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t max_repairs,
                              int32_t max_lifts, int32_t flags, int32_t algo, int32_t* commit_read,
                              int32_t* lookup_read, jtb_lk_shard* shards, jtb_lk_result* out) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (algo != LK_SEARCH && algo != LK_BRUTE) { g_err = "unknown algorithm"; return -2; }
    const int32_t NS = h->n_shards;
    memset(out, 0, sizeof *out);
    if (algo == LK_BRUTE) {
        int64_t n_records = 0;
        for (int32_t s = 0; s < NS; ++s) {
            Shard S;
            if (int rc = parse_shard(h, s, S, n_records)) return rc;
            jtb_lk_shard& o = shards[s];
            memset(&o, 0, sizeof o);
            const int v = brute_shard(S, parse_lookups(h, s));
            if (v < 0) { g_err = "LK_BRUTE: a shard has more than 24 ops"; return -2; }
            o.valid = v ? JTB_VALID : JTB_INVALID;
            o.n_reads = (int32_t)S.R.size();
            o.n_transfers = (int32_t)S.T.size();
            out->valid = std::max(out->valid, o.valid);
        }
        return 0;
    }
    std::vector<jtb_cw_shard> cw(std::max(NS, 1));
    jtb_cw_result cr;
    int64_t nT = 0;
    for (int32_t s = 0; s < NS; ++s) {
        Shard S;
        int64_t n_records = 0;
        if (int rc = parse_shard(h, s, S, n_records)) return rc;
        nT += (int64_t)S.T.size();
    }
    std::vector<int32_t> commit(std::max<int64_t>(nT, 1));
    if (int rc = jtbm_check_class_witness(h, max_nodes, max_rounds, max_repairs, max_lifts, 0, 1, commit.data(),
                                          cw.data(), &cr)) {
        g_err = jtbm_cw_last_error();
        return rc;
    }
    int64_t at = 0, lat = 0;
    for (int32_t s = 0; s < NS; ++s) {
        Shard S;
        int64_t n_records = 0;
        if (int rc = parse_shard(h, s, S, n_records)) return rc;
        const std::vector<LLookup> L = parse_lookups(h, s);
        jtb_lk_shard& o = shards[s];
        memset(&o, 0, sizeof o);
        const jtb_cw_shard& c = cw[s];
        o.valid = c.valid; o.cause = c.cause; o.n_reads = c.n_reads; o.n_transfers = c.n_transfers;
        o.n_committed = c.n_committed; o.n_committed_crashed = c.n_committed_crashed; o.n_after = c.n_after;
        o.nodes = c.nodes; o.rounds = c.rounds; o.fail_index = c.fail_index; o.transfer_id = c.transfer_id;
        o.repairs = c.repairs; o.n_bans = c.n_bans; o.lifts = c.lifts; o.n_lifted = c.n_lifted;
        o.class_cause = c.class_cause; o.class_rounds = c.class_rounds; o.n_handed = c.n_handed;
        o.lookup_fail_index = -1;
        std::vector<int32_t> cm(commit.begin() + at, commit.begin() + at + (int64_t)S.T.size());
        std::vector<int32_t> lr(L.size(), JTB_SW_NEVER);
        if (o.valid == JTB_VALID && !L.empty()) {
            classify_inputs(S);
            std::vector<int32_t> keys, ord;
            bool partial;
            shard_order(S, keys, partial, ord);
            lookup_pass(S, ord, L, o, cm, lr);
        }
        if (commit_read) std::copy(cm.begin(), cm.end(), commit_read + at);
        if (lookup_read) std::copy(lr.begin(), lr.end(), lookup_read + lat);
        at += (int64_t)S.T.size();
        lat += (int64_t)L.size();
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_committed += o.n_committed;
        out->n_committed_crashed += o.n_committed_crashed;
        out->n_after += o.n_after;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
        out->repairs = std::max(out->repairs, (int64_t)o.repairs);
        out->n_bans += o.n_bans;
        out->lifts = std::max(out->lifts, (int64_t)o.lifts);
        out->n_lifted += o.n_lifted;
        out->class_rounds = std::max(out->class_rounds, (int64_t)o.class_rounds);
        out->n_handed += o.n_handed;
        out->n_lookups_placed += o.n_lookups_placed;
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
