// class_witness.cpp — CPU oracle of the class witness (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// CW_SEARCH is the library's decision, shard by shard: LW_SEARCH, then a class pass on every shard LW_SEARCH leaves
// UNKNOWN with cause UNDECIDED, NO_WITNESS or REAL_TIME (DESIGN.md "K16 class witness").  The class pass starts from
// TP_SEARCH's owners: the crashed transfers with a window that no gap owns fall into classes by (debit, credit, amount,
// M(t), A(t)), each ordered by (invocation, id); witness rounds gather with at most cap members per class (gaps_common.h)
// and keep, per class, how many members they chose; the gaps of a round then receive members by rank in gap order, and a
// gap is fixed when no smaller gap took one of its :ok transfers, every member it received exists and is eligible for
// it, and no gap of the round up to it that draws from one of its classes failed that.  The witness's real-time pass
// and re-sum decide.  Node counts, rounds, class rounds and the members handed out are the library's.
#include <map>
#include <tuple>

#include "repair_common.h"

namespace {

constexpr int CW_SEARCH = 1;

void roll_cw(jtb_cw_result* out, const jtb_cw_shard& o) {
    out->lifts = std::max(out->lifts, (int64_t)o.lifts);
    out->n_lifted += o.n_lifted;
    out->class_rounds = std::max(out->class_rounds, (int64_t)o.class_rounds);
    out->n_handed += o.n_handed;
}

// the class pass on one shard, from TP_SEARCH's state T; a shard it proves becomes VALID with its counts and commit_read
int class_pass(const Shard& S, const std::vector<int32_t>& keys, const std::vector<int32_t>& ord, TpState& T,
               int64_t max_nodes, int32_t max_rounds, RepairOut<jtb_cw_shard>& w) {
    jtb_cw_shard& o = w.o;
    Witness x(S, keys, ord, T);
    const int32_t n = x.n, K = x.K, nT = x.nT;
    std::vector<int32_t>& owner = T.owner;
    // the classes and their members by (invocation, id)
    std::map<std::tuple<int32_t, int32_t, int32_t, int32_t, int32_t>, int32_t> class_of;
    std::vector<int32_t> cls(nT, -1);
    std::vector<std::vector<int32_t>> members;
    for (int32_t t = 0; t < nT; ++t) {
        const XTransfer& z = S.T[t];
        if (z.fate == JTB_T_OK || !T.W[t].win || owner[t] >= 0) continue;
        auto it = class_of.emplace(std::make_tuple(z.debit, z.credit, z.amount, z.M, z.A), (int32_t)members.size());
        if (it.second) members.emplace_back();
        cls[t] = it.first->second;
        members[cls[t]].push_back(t);
    }
    for (auto& c : members)
        std::sort(c.begin(), c.end(), [&](int32_t a, int32_t b) {
            return S.T[a].inv != S.T[b].inv ? S.T[a].inv < S.T[b].inv : S.T[a].id < S.T[b].id;
        });
    auto eligible = [&](int32_t t, int32_t i) {
        const XTransfer& z = S.T[t];
        const XRead& u = x.upper(i);
        return T.W[t].win && T.W[t].lo <= i && i <= T.W[t].hi && z.inv < u.comp && z.A < u.comp &&
               !(z.M < (x.lower(i) ? x.lower(i)->inv : -1));
    };
    int32_t failed = -1, rounds = 0;
    int64_t handed = 0;
    for (int32_t round = 0;; ++round) {
        int32_t first = -1;
        for (int32_t i = 0; i < n && first < 0; ++i)
            if (!x.fixed[i]) first = i;
        if (first < 0) break;
        if (round >= max_rounds) { failed = first; break; }
        rounds++;
        // the searches: the chosen :ok transfers and the chosen crashed ones (members of their class)
        std::vector<std::vector<int32_t>> okc(n), crc(n);
        for (int32_t i = 0; i < n; ++i) {
            if (x.fixed[i]) continue;
            Problem pb;
            pb.key = keys;
            pb.d.resize(K);
            bool neg = false;
            for (int32_t j = 0; j < K; ++j) neg |= (pb.d[j] = x.delta(i, j)) < 0;
            bool ok = !neg && gather_gap(S, x.X, T.W, owner, x.upper(i), x.lower(i), i, 1, pb, nullptr, &cls);
            if (ok) {
                Search s(pb, -1, max_nodes);
                int32_t root_key, kept;
                std::vector<uint8_t> sol;
                ok = s.run(root_key, kept, nullptr, nullptr, &sol) == EXPLAINED;
                o.nodes += s.nodes;
                if (ok)
                    for (size_t c = 0; c < pb.P.size(); ++c)
                        if (sol[c] == IN) (S.T[pb.P[c].t].fate == JTB_T_OK ? okc : crc)[i].push_back(pb.P[c].t);
            }
            if (!ok && failed < 0) failed = i;
        }
        if (failed >= 0) break;
        // K13's rule for the :ok transfers
        std::vector<int32_t> cmin(nT, INT_MAX);
        for (int32_t i = 0; i < n; ++i)
            for (int32_t t : okc[i]) cmin[t] = std::min(cmin[t], i);
        std::vector<char> ok1(n, 1);
        for (int32_t i = 0; i < n; ++i)
            for (int32_t t : okc[i]) ok1[i] &= cmin[t] == i;
        // the hand-out: per class, ranks in gap order over the unowned members
        std::vector<std::vector<int32_t>> un(members.size());
        for (size_t c = 0; c < members.size(); ++c)
            for (int32_t t : members[c])
                if (owner[t] < 0) un[c].push_back(t);
        std::vector<size_t> next(members.size(), 0);
        std::vector<int32_t> cfail(members.size(), INT_MAX);
        std::vector<std::vector<int32_t>> got(n);
        for (int32_t i = 0; i < n; ++i)
            for (int32_t t : crc[i]) {
                const int32_t c = cls[t];
                const size_t r = next[c]++;
                if (ok1[i] && r < un[c].size() && eligible(un[c][r], i)) got[i].push_back(un[c][r]);
                else cfail[c] = std::min(cfail[c], i);
            }
        for (int32_t i = 0; i < n; ++i) {
            if (x.fixed[i]) continue;
            bool fix = ok1[i];
            for (int32_t t : crc[i]) fix &= i < cfail[cls[t]];
            if (!fix) continue;
            x.fixed[i] = 1;
            for (int32_t t : okc[i]) owner[t] = i;
            for (int32_t t : got[i]) owner[t] = i;
            handed += (int64_t)got[i].size();
        }
    }
    o.class_rounds = rounds;
    o.n_handed = handed;
    if (failed >= 0) {
        o.class_cause = JTB_CAUSE_NO_WITNESS;
        return 0;
    }
    if (!x.check()) {
        g_err = "the counters of a serial witness do not add up";
        return -1;
    }
    jtb_cw_shard v = o;
    v.valid = JTB_VALID;
    v.cause = 0;
    v.fail_index = -1;
    v.transfer_id = -1;
    v.n_committed = v.n_committed_crashed = v.n_after = 0;
    std::vector<int32_t> commit(nT, JTB_SW_NEVER);
    x.verdict(v, commit);
    if (v.valid != JTB_VALID) {
        o.class_cause = JTB_CAUSE_REAL_TIME;
        return 0;
    }
    o = v;
    w.commit = commit;
    return 0;
}

}  // namespace

extern "C" {

const char* jtbm_cw_last_error(void) { return g_err.c_str(); }

int jtbm_check_class_witness(const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t max_repairs,
                             int32_t max_lifts, int32_t flags, int32_t algo, int32_t* commit_read,
                             jtb_cw_shard* shards, jtb_cw_result* out) {
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (algo != CW_SEARCH) { g_err = "unknown algorithm"; return -2; }
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    return repaired_check(h, max_nodes, max_rounds, max_repairs, max_lifts, commit_read, shards, out, roll_cw,
                          class_pass);
}

}  // extern "C"
