// repair_common.h — the repair loop and the per-shard driver that RW_SEARCH and LW_SEARCH share (TEST INFRASTRUCTURE
// ONLY).  RW_SEARCH runs it with no lift steps (max_lifts 0): a repair that records no new ban ends the shard.
// LW_SEARCH runs a lift step there instead (DESIGN.md "K15 lifted serial witness"): the failing gaps steal again with
// their own bans ignored and P^0 (the reads' invocations alone) in place of P^; a kept thief's bans on its loot are
// lifted, and the repairs resume.  Node counts, rounds, repairs, bans and lifts are the library's.
#pragma once
#include <chrono>
#include <cstring>
#include <set>

#include "witness_common.h"

namespace {

template <class O>
struct RepairOut {
    O o;
    std::vector<int32_t> commit;   // per transfer of the shard
};

inline void set_lifts(jtb_rw_shard&, int32_t, int32_t) {}
inline void set_lifts(jtb_lw_shard& o, int32_t lifts, int32_t n_lifted) {
    o.lifts = lifts;
    o.n_lifted = n_lifted;
}
inline void set_lifts(jtb_cw_shard& o, int32_t lifts, int32_t n_lifted) {
    o.lifts = lifts;
    o.n_lifted = n_lifted;
}

// the steals of the failing gaps (Jacobi): gap g searches the free and the chosen transfers that keep(t, g) admits; a
// thief keeps its solution when no smaller thief took one of them.  thief, loot and rel (every failing gap) per gap
template <class O>
void steals(Witness& x, int64_t max_nodes, const std::function<bool(int32_t, int32_t)>& keep, O& o,
            std::vector<char>& thief, std::vector<std::vector<int32_t>>& loot, std::vector<char>& rel) {
    const int32_t nT = x.nT;
    std::vector<int32_t> free_(x.T.owner), cmin(nT, INT_MAX);
    for (int32_t t = 0; t < nT; ++t)
        if (x.chosen_t(t)) free_[t] = -1;
    for (int32_t g : x.failing) {
        rel[g] = 1;
        const std::function<bool(int32_t)> k = [&](int32_t t) { return keep(t, g); };
        Problem pb;
        if (!x.gather(g, free_, &k, pb)) continue;
        Search sr(pb, -1, max_nodes);
        int32_t root_key, kept;
        std::vector<uint8_t> sol;
        const bool ok = sr.run(root_key, kept, nullptr, nullptr, &sol) == EXPLAINED;
        o.nodes += sr.nodes;
        if (!ok) continue;
        thief[g] = 1;
        for (size_t c = 0; c < pb.P.size(); ++c)
            if (sol[c] == IN) {
                loot[g].push_back(pb.P[c].t);
                cmin[pb.P[c].t] = std::min(cmin[pb.P[c].t], g);
            }
    }
    for (int32_t g : x.failing)
        for (int32_t t : loot[g]) thief[g] &= cmin[t] == g;
}

// the witness of a shard TP_SEARCH called VALID, then repairs (and, with max_lifts > 0, lift steps) until it is proved
// or they stop
template <class O>
int repaired(const Shard& S, const std::vector<int32_t>& keys, const std::vector<int32_t>& ord, TpState& T,
             int64_t max_nodes, int32_t max_rounds, int32_t max_repairs, int32_t max_lifts, RepairOut<O>& w) {
    O& o = w.o;
    Witness x(S, keys, ord, T);
    const int32_t n = x.n, nT = x.nT;
    std::vector<int32_t>& owner = T.owner;
    std::set<std::pair<int32_t, int32_t>> bans;     // (gap, transfer) banned now
    std::set<std::pair<int32_t, int32_t>> lifted;   // (gap, transfer) lifted once
    int32_t n_bans = 0, lifts = 0, n_lifted = 0;
    std::vector<int32_t> Ph(n), P0(n);              // P^ and P^0 at each position
    auto hat = [&]() {
        std::vector<int32_t> gmax(n, INT_MIN);
        for (int32_t t = 0; t < nT; ++t)
            if (owner[t] >= 0) gmax[owner[t]] = std::max(gmax[owner[t]], S.T[t].inv);
        for (int32_t i = 0; i < n; ++i) Ph[i] = std::max({i > 0 ? Ph[i - 1] : INT_MIN, x.upper(i).inv, gmax[i]});
    };
    for (int32_t i = 0; i < n; ++i) P0[i] = std::max(i > 0 ? P0[i - 1] : INT_MIN, x.upper(i).inv);
    auto keep = [&](int32_t t, int32_t i) { return !bans.count({i, t}) && !(i > 0 && S.T[t].okcomp <= Ph[i - 1]); };
    // a lift step's gather: g's own bans ignored unless lifted before, and P^0 in place of P^
    auto lift_keep = [&](int32_t t, int32_t i) {
        return !(bans.count({i, t}) && lifted.count({i, t})) && !(i > 0 && S.T[t].okcomp <= P0[i - 1]);
    };
    for (int32_t rep = 0;; ++rep) {
        int32_t rounds = 0;
        const int32_t failed = rep ? x.rounds(max_nodes, max_rounds, hat, keep, rounds, o.nodes)
                                   : x.rounds(max_nodes, max_rounds, {}, {}, rounds, o.nodes);
        o.rounds += rounds;
        o.valid = JTB_VALID;
        o.cause = 0;
        o.fail_index = -1;
        o.transfer_id = -1;
        if (failed >= 0) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_NO_WITNESS;
            o.fail_index = x.upper(failed).comp_index;
        } else {
            if (!x.check()) {
                g_err = "the counters of a serial witness do not add up";
                return -1;
            }
            x.verdict(o, w.commit);
            if (o.valid == JTB_VALID) return 0;
        }
        if (rep >= max_repairs + (lifts ? max_lifts : 0)) return 0;
        // the blame: new bans, and the gaps they release
        std::vector<std::pair<int32_t, int32_t>> nb;
        std::vector<char> rel(n, 0), thief(n, 0);
        std::vector<std::vector<int32_t>> loot(n);
        hat();
        auto take = [&]() {   // the bans of the chosen transfers in the kept thieves' loot
            for (int32_t g : x.failing)
                if (thief[g])
                    for (int32_t t : loot[g])
                        if (x.chosen_t(t)) nb.push_back({owner[t], t});
        };
        if (failed >= 0) {
            steals(x, max_nodes, keep, o, thief, loot, rel);
            take();
        } else {
            // real time: every chosen transfer of D_g that completes by P_g, and every chosen transfer of a gap h
            // invoked at or after SM[h], the smallest completion of what must follow it (the reads from r_h on, D_g
            // for g > h, the failing :ok transfers after the last read)
            int32_t after = INT_MAX;
            for (int32_t t = 0; t < nT; ++t)
                if (x.after_fails(t)) after = std::min(after, S.T[t].okcomp);
            std::vector<int32_t> SM(n + 1);
            SM[n] = after;
            for (int32_t i = n - 1; i >= 0; --i)
                SM[i] = std::min({SM[i + 1], x.upper(i).comp, i + 1 < n ? x.gmin[i + 1] : INT_MAX});
            for (int32_t t = 0; t < nT; ++t) {
                if (!x.chosen_t(t)) continue;
                const int32_t g = owner[t];
                if ((g > 0 && S.T[t].okcomp <= x.Q[g - 1]) || S.T[t].inv >= SM[g]) nb.push_back({g, t});
            }
        }
        if (nb.empty()) {
            // the lift step: only after a NO_WITNESS repair, within the budget, and only when it lifts a ban
            if (failed < 0 || lifts >= max_lifts) return 0;
            std::fill(rel.begin(), rel.end(), 0);
            std::fill(thief.begin(), thief.end(), 0);
            for (auto& l : loot) l.clear();
            steals(x, max_nodes, lift_keep, o, thief, loot, rel);
            int32_t nl = 0;
            for (int32_t g : x.failing)
                if (thief[g])
                    for (int32_t t : loot[g])
                        if (bans.erase({g, t})) {
                            lifted.insert({g, t});
                            nl++;
                        }
            if (!nl) return 0;
            take();
            lifts++;
            n_lifted += nl;
        }
        for (auto& p : nb) {
            bans.insert(p);
            rel[p.first] = 1;
        }
        n_bans += (int32_t)nb.size();
        o.repairs = rep + 1;
        o.n_bans = n_bans;
        set_lifts(o, lifts, n_lifted);
        for (int32_t i = 0; i < n; ++i)
            if (rel[i]) x.fixed[i] = 0;
        for (int32_t t = 0; t < nT; ++t)
            if (x.chosen_t(t) && rel[owner[t]]) owner[t] = -1;
        for (int32_t g = 0; g < n; ++g)
            if (thief[g]) {
                x.fixed[g] = 1;
                for (int32_t t : loot[g]) owner[t] = g;
            }
    }
}

// every shard of h: the witness and its repairs where TP_SEARCH calls the shard VALID; O / R the shard and result
// structs (jtb_rw_*, jtb_lw_* or jtb_cw_*).  post (may be null) runs on every shard that ends UNKNOWN with cause
// UNDECIDED, NO_WITNESS or REAL_TIME, with TP_SEARCH's state as TP_SEARCH left it
template <class O, class R>
int repaired_check(const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t max_repairs,
                   int32_t max_lifts, int32_t* commit_read, O* shards, R* out,
                   void (*roll)(R*, const O&),
                   int (*post)(const Shard&, const std::vector<int32_t>&, const std::vector<int32_t>&, TpState&,
                               int64_t, int32_t, RepairOut<O>&) = nullptr) {
    const auto t0 = std::chrono::steady_clock::now();
    if (max_nodes <= 0) max_nodes = JTB_TP_DEFAULT_MAX_NODES;
    if (max_rounds <= 0) max_rounds = JTB_TP_DEFAULT_MAX_ROUNDS;
    if (max_repairs <= 0) max_repairs = JTB_RW_DEFAULT_MAX_REPAIRS;
    memset(out, 0, sizeof *out);
    int64_t n_records = 0, n_reads = 0;
    std::vector<RepairOut<O>> tmp(h->n_shards);
    try {
        for (int32_t s = 0; s < h->n_shards; ++s) {
            Shard S;
            if (int rc = parse_shard(h, s, S, n_records)) return rc;
            n_reads += (int64_t)S.R.size();
            if (n_reads > INT_MAX) { g_err = "more than 2^31-1 reads"; return -2; }
            classify_inputs(S);
            RepairOut<O>& w = tmp[s];
            O& o = w.o;
            memset(&o, 0, sizeof o);
            o.valid = JTB_VALID;
            o.n_reads = (int32_t)S.R.size();
            o.n_transfers = (int32_t)S.T.size();
            o.fail_index = -1;
            o.transfer_id = -1;
            w.commit.assign(S.T.size(), JTB_SW_NEVER);
            std::vector<int32_t> keys, ord;
            bool partial;
            shard_order(S, keys, partial, ord);
            if (partial) {
                o.valid = JTB_UNKNOWN;
                o.cause = JTB_CAUSE_PARTIAL_READ;
                continue;
            }
            if (S.R.empty()) {
                for (size_t t = 0; t < S.T.size(); ++t)
                    if (S.T[t].fate == JTB_T_OK) w.commit[t] = JTB_SW_FREE;
                continue;
            }
            jtb_tp_shard p;
            memset(&p, 0, sizeof p);
            TpState T;
            tp_search(h, s, S, keys, ord, max_nodes, max_rounds, p, T);
            if (p.valid != JTB_VALID) {
                o.valid = JTB_UNKNOWN;
                o.cause = p.valid == JTB_INVALID ? JTB_CAUSE_ANOMALY : JTB_CAUSE_UNDECIDED;
                if (post && o.cause == JTB_CAUSE_UNDECIDED)
                    if (int rc = post(S, keys, ord, T, max_nodes, max_rounds, w)) return rc;
                continue;
            }
            TpState T0;
            if (post) T0 = T;
            if (int rc = repaired(S, keys, ord, T, max_nodes, max_rounds, max_repairs, max_lifts, w)) return rc;
            if (o.valid != JTB_VALID) {
                o.n_committed = o.n_committed_crashed = o.n_after = 0;
                std::fill(w.commit.begin(), w.commit.end(), JTB_SW_NEVER);
                if (post)
                    if (int rc = post(S, keys, ord, T0, max_nodes, max_rounds, w)) return rc;
            }
        }
    } catch (int) {
        return -2;
    }
    int64_t at = 0;
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const O& o = shards[s] = tmp[s].o;
        if (commit_read) std::copy(tmp[s].commit.begin(), tmp[s].commit.end(), commit_read + at);
        at += (int64_t)tmp[s].commit.size();
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_committed += o.n_committed;
        out->n_committed_crashed += o.n_committed_crashed;
        out->n_after += o.n_after;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
        out->repairs = std::max(out->repairs, (int64_t)o.repairs);
        out->n_bans += o.n_bans;
        roll(out, o);
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // namespace
