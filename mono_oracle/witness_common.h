// witness_common.h — the witness of the serial-witness check on one shard, which SW_SEARCH and RW_SEARCH share (TEST
// INFRASTRUCTURE ONLY): the witness rounds, the re-sum of the counters, the greedy real-time pass and commit_read.  The
// repaired witness adds a filter to the rounds' gather and re-runs them; the serial-witness check runs them once.
#pragma once
#include <functional>

#include "gaps_common.h"

namespace {

// the witness of one shard TP_SEARCH called VALID; T's owners become the witness's D_g
struct Witness {
    const Shard& S;
    const std::vector<int32_t>& keys;
    const std::vector<int32_t>& ord;
    TpState& T;
    const Index X;
    const int32_t n, K, nT;
    std::vector<int32_t> kowner;              // the owners TP_SEARCH left (the witness never releases them)
    std::vector<char> fixed;
    std::vector<std::vector<int32_t>> chosen;
    std::vector<int32_t> failing;             // of the last rounds: the gaps the failing round did not explain, or
                                              // every unfixed gap when max_rounds ran out
    // of the last real-time pass: Q[i] = the point of the read at position i, D_g's largest invocation and smallest
    // :ok completion, the failure key (position << 1 | 1: read, 0: transfer), ~0 none
    std::vector<int32_t> Q, gmax, gmin;
    uint64_t best = ~0ull;

    Witness(const Shard& S_, const std::vector<int32_t>& keys_, const std::vector<int32_t>& ord_, TpState& T_)
        : S(S_), keys(keys_), ord(ord_), T(T_), X(S_, keys_), n((int32_t)ord_.size()), K((int32_t)keys_.size()),
          nT((int32_t)S_.T.size()), kowner(T_.owner), fixed(n, 1), chosen(n) {
        for (int32_t i = 0; i < n; ++i)
            for (int32_t j = 0; j < K; ++j) fixed[i] &= delta(i, j) == 0;
    }

    const XRead& upper(int32_t i) const { return S.R[ord[i]]; }
    const XRead* lower(int32_t i) const { return i > 0 ? &S.R[ord[i - 1]] : nullptr; }
    int64_t delta(int32_t i, int32_t j) const {
        return upper(i).kv[j].second - (lower(i) ? lower(i)->kv[j].second : 0) - T.G[i].own[j];
    }
    // a chosen transfer: owned by a gap, and not by TP_SEARCH
    bool chosen_t(int32_t t) const { return T.owner[t] >= 0 && kowner[t] < 0; }

    // gap i's gather with `keep` (nullptr: none) as an extra filter; false: the gather passed the cap or Delta' < 0
    bool gather(int32_t i, const std::vector<int32_t>& owner, const std::function<bool(int32_t)>* keep,
                Problem& pb) const {
        pb.key = keys;
        pb.d.resize(K);
        bool neg = false;
        for (int32_t j = 0; j < K; ++j) neg |= (pb.d[j] = delta(i, j)) < 0;
        return !neg && gather_gap(S, X, T.W, owner, upper(i), lower(i), i, 1, pb, keep);
    }

    // the witness rounds over the unfixed gaps (Jacobi); before (may be empty) runs at the start of every round, and
    // keep(t, i) (may be empty) filters gap i's gather.  The failing gap (the first a round did not explain, else the
    // first unfixed one when max_rounds ran out), -1 none; all of them into failing
    int32_t rounds(int64_t max_nodes, int32_t max_rounds, const std::function<void()>& before,
                   const std::function<bool(int32_t, int32_t)>& keep, int32_t& n_rounds, int64_t& nodes) {
        failing.clear();
        for (int32_t round = 0;; ++round) {
            int32_t first = -1;
            for (int32_t i = 0; i < n && first < 0; ++i)
                if (!fixed[i]) first = i;
            if (first < 0) return -1;
            if (round >= max_rounds) {
                for (int32_t i = 0; i < n; ++i)
                    if (!fixed[i]) failing.push_back(i);
                return first;
            }
            n_rounds++;
            if (before) before();
            int32_t failed = -1;
            for (int32_t i = 0; i < n; ++i) {
                if (fixed[i]) continue;
                chosen[i].clear();
                Problem pb;
                const std::function<bool(int32_t)> k = [&](int32_t t) { return keep(t, i); };
                bool ok = gather(i, T.owner, keep ? &k : nullptr, pb);
                if (ok) {
                    Search s(pb, -1, max_nodes);
                    int32_t root_key, kept;
                    std::vector<uint8_t> sol;
                    ok = s.run(root_key, kept, nullptr, nullptr, &sol) == EXPLAINED;
                    nodes += s.nodes;
                    if (ok)
                        for (size_t c = 0; c < pb.P.size(); ++c)
                            if (sol[c] == IN) chosen[i].push_back(pb.P[c].t);
                }
                if (!ok) failing.push_back(i);
                if (!ok && failed < 0) failed = i;
            }
            if (failed >= 0) return failed;
            std::vector<int32_t> cmin(nT, INT_MAX);
            for (int32_t i = 0; i < n; ++i)
                if (!fixed[i])
                    for (int32_t t : chosen[i]) cmin[t] = std::min(cmin[t], i);
            std::vector<char> fix(n, 0);
            for (int32_t i = 0; i < n; ++i) {
                if (fixed[i]) continue;
                fix[i] = 1;
                for (int32_t t : chosen[i]) fix[i] &= cmin[t] == i;
            }
            for (int32_t i = 0; i < n; ++i)
                if (fix[i]) {
                    fixed[i] = 1;
                    for (int32_t t : chosen[i]) T.owner[t] = i;
                }
        }
    }

    // the counters of every gap summed from D_g (false: they do not add up), then the real-time pass into Q, gmax,
    // gmin and best
    bool check() {
        const std::vector<int32_t>& owner = T.owner;
        std::vector<std::vector<int64_t>> sum(n, std::vector<int64_t>(K, 0));
        for (int32_t t = 0; t < nT; ++t) {
            if (owner[t] < 0) continue;
            if (T.W[t].jd >= 0) sum[owner[t]][T.W[t].jd] += S.T[t].amount;
            if (T.W[t].jc >= 0) sum[owner[t]][T.W[t].jc] += S.T[t].amount;
        }
        for (int32_t i = 0; i < n; ++i)
            for (int32_t j = 0; j < K; ++j)
                if (sum[i][j] != upper(i).kv[j].second - (lower(i) ? lower(i)->kv[j].second : 0)) return false;
        gmax.assign(n, INT_MIN);
        gmin.assign(n, INT_MAX);
        for (int32_t t = 0; t < nT; ++t) {
            if (owner[t] < 0) continue;
            gmax[owner[t]] = std::max(gmax[owner[t]], S.T[t].inv);
            gmin[owner[t]] = std::min(gmin[owner[t]], S.T[t].okcomp);
        }
        Q.assign(n, 0);
        best = ~0ull;
        for (int32_t i = 0; i < n; ++i) {
            Q[i] = std::max({i > 0 ? Q[i - 1] : INT_MIN, upper(i).inv, gmax[i]});
            if (i > 0 && gmin[i] <= Q[i - 1]) best = std::min(best, (uint64_t)i << 1);
            if (Q[i] >= upper(i).comp) best = std::min(best, (uint64_t)i << 1 | 1);
        }
        for (int32_t t = 0; t < nT; ++t)
            if (after_fails(t)) best = std::min(best, (uint64_t)n << 1);
        return true;
    }

    // an :ok transfer with a window in no D_g that completed before the last read's point
    bool after_fails(int32_t t) const {
        return S.T[t].fate == JTB_T_OK && T.W[t].win && T.owner[t] < 0 && S.T[t].okcomp <= Q[n - 1];
    }
    // a transfer that fails at the real-time failure key `best` (a transfer failure)
    bool rt_fails(int32_t t) const {
        const int32_t at = (int32_t)(best >> 1);
        return at < n ? T.owner[t] == at && S.T[t].okcomp <= Q[at - 1] : after_fails(t);
    }

    // the verdict of the last check into o (cause, fail_index, transfer_id), and commit_read when it is VALID
    template <class O>
    void verdict(O& o, std::vector<int32_t>& commit) const {
        if (best != ~0ull) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_REAL_TIME;
            const int32_t at = (int32_t)(best >> 1);
            if (best & 1) {
                o.fail_index = upper(at).comp_index;
                return;
            }
            int32_t wt = -1;
            for (int32_t t = 0; t < nT; ++t)
                if (rt_fails(t) && (wt < 0 || S.T[t].id < S.T[wt].id)) wt = t;
            o.fail_index = S.T[wt].cidx;
            o.transfer_id = S.T[wt].id;
            return;
        }
        for (int32_t t = 0; t < nT; ++t) {
            const XTransfer& x = S.T[t];
            if (T.owner[t] >= 0) {
                commit[t] = upper(T.owner[t]).comp_index;
                o.n_committed++;
                o.n_committed_crashed += x.fate != JTB_T_OK;
            } else if (x.fate == JTB_T_OK && T.W[t].win) {
                commit[t] = JTB_SW_AFTER;
                o.n_after++;
            } else if (x.fate == JTB_T_OK) {
                commit[t] = JTB_SW_FREE;
            }
        }
    }
};

}  // namespace
