// transfer_placement.cpp — CPU oracle of the transfer-placement check (TEST INFRASTRUCTURE ONLY; the library never
// calls it).
//
// Both deciders parse a shard, order its reads and form its gaps as the read-gap oracle does (gaps_common.h), give
// every transfer its window of gaps [lo, hi] and fill jtb_tp_shard as jtb_check_transfer_placement does.
// TP_BRUTE is the definition: every assignment of each windowed transfer to one gap of its window, or to none for a
// may transfer, and whether some assignment makes every gap sum to Delta on every key.  No caps; tiny histories only.
// TP_SEARCH is the library's: round 0 is RG_SEARCH gap for gap, then the owner / PLACE / LOST pass after every round,
// the re-runs of round 1 (every gap) and of the dirtied gaps after it with Delta' and the in-window gather, the latch
// and the witness.  Node counts and rounds are the library's.
#include <chrono>
#include <cstring>
#include <memory>

#include "gaps_common.h"

namespace {

constexpr int TP_BRUTE = 0, TP_SEARCH = 1;

// a transfer's window of gaps; win: the transfer is not :fail, has a positive amount and touches an observed key
struct Window {
    bool win = false, must = false;
    int32_t lo = 0, hi = -1, jd = -1, jc = -1;
};

std::vector<Window> windows(const Shard& S, const std::vector<int32_t>& keys, const std::vector<int32_t>& ord) {
    const int32_t n = (int32_t)ord.size();
    std::vector<int32_t> pos(n), pmax(n), by_inv(n), smin(n + 1, INT_MAX);
    for (int32_t i = 0; i < n; ++i) pos[ord[i]] = i;
    for (int32_t r = 0; r < n; ++r) pmax[r] = std::max(r ? pmax[r - 1] : -1, pos[r]);   // S.R: completion order
    for (int32_t r = 0; r < n; ++r) by_inv[r] = r;
    std::stable_sort(by_inv.begin(), by_inv.end(), [&](int32_t a, int32_t b) { return S.R[a].inv < S.R[b].inv; });
    for (int32_t k = n - 1; k >= 0; --k) smin[k] = std::min(smin[k + 1], pos[by_inv[k]]);
    std::vector<int32_t> comp(n), inv(n);
    for (int32_t r = 0; r < n; ++r) {
        comp[r] = S.R[r].comp;
        inv[r] = S.R[by_inv[r]].inv;
    }
    std::vector<Window> W(S.T.size());
    for (size_t t = 0; t < S.T.size(); ++t) {
        const XTransfer& x = S.T[t];
        Window& w = W[t];
        w.jd = col_of(keys, 2 * (int64_t)x.debit);
        w.jc = col_of(keys, 2 * (int64_t)x.credit + 1);
        if (x.fate == JTB_T_FAIL || x.amount <= 0 || (w.jd < 0 && w.jc < 0) || n == 0) continue;
        w.win = true;
        // lo: past every read that completed before max(iv(t), A(t)); hi: the first read (in the order) invoked after M
        const int32_t cut = std::max(x.inv, x.A);
        const int32_t c = (int32_t)(std::lower_bound(comp.begin(), comp.end(), cut) - comp.begin());
        w.lo = c ? pmax[c - 1] + 1 : 0;
        const int32_t k = (int32_t)(std::upper_bound(inv.begin(), inv.end(), x.M) - inv.begin());
        w.must = k < n;
        w.hi = w.must ? smin[k] : n - 1;
    }
    return W;
}

// ---- TP_BRUTE ----------------------------------------------------------------------------------------------------
struct Brute {
    const Shard& S;
    const std::vector<Window>& W;
    std::vector<std::vector<int64_t>> need;   // per gap, per key: what is left of Delta
    std::vector<int32_t> ts;
    int64_t leaves = 0;

    bool put(int32_t t, int32_t g, int sign) {
        const Window& w = W[t];
        const int64_t a = sign * (int64_t)S.T[t].amount;
        bool ok = true;
        if (w.jd >= 0) ok &= (need[g][w.jd] -= a) >= 0;
        if (w.jc >= 0) ok &= (need[g][w.jc] -= a) >= 0;
        return ok;
    }
    bool go(size_t j) {
        if (j == ts.size()) {
            if (++leaves > (1 << 22)) { g_err = "TP_BRUTE: more than 2^22 assignments"; throw 1; }
            for (auto& v : need)
                for (int64_t x : v)
                    if (x != 0) return false;
            return true;
        }
        const int32_t t = ts[j];
        if (!W[t].must && go(j + 1)) return true;
        for (int32_t g = W[t].lo; g <= W[t].hi; ++g) {
            const bool ok = put(t, g, 1);
            const bool found = ok && go(j + 1);
            put(t, g, -1);
            if (found) return true;
        }
        return false;
    }
};

// ---- TP_SEARCH ---------------------------------------------------------------------------------------------------
struct Gap {
    int8_t code = G_EXPLAINED;     // of the last round that ran the gap
    int8_t lcode = 0;              // the latched unexplained kind, 0 none
    int32_t lround = -1, lkey = -1, kept = 0;
    int64_t ldelta = 0;
    bool inc = false;              // the gather passed the cap, or the shard has too many keys
    std::vector<int32_t> poss;     // transfers gathered and not pruned out by the root
    std::vector<int32_t> forced;   // this round
    std::vector<int64_t> own;      // per key: the amounts of the transfers the gap owns
};

// one run of gap i (upper read u, lower read l) in round `round`
void run_gap(const Shard& S, const std::vector<int32_t>& keys, const Index& X, const std::vector<Window>& W,
             const std::vector<int32_t>& owner, const XRead& u, const XRead* l, int32_t i, int32_t round,
             int64_t max_nodes, int64_t& nodes, Gap& g) {
    const int32_t K = (int32_t)keys.size();
    g.poss.clear();
    g.forced.clear();
    g.inc = false;
    g.kept = 0;
    int8_t code = G_EXPLAINED;
    int32_t key = -1;
    int64_t delta = 0;
    auto latch = [&]() {
        g.code = code;
        if (code != G_EXPLAINED && code != G_UNDECIDED && !g.lcode) {
            g.lcode = code;
            g.lround = round;
            g.lkey = key;
            g.ldelta = delta;
        }
    };
    if (K > JTB_TP_MAX_KEYS) { code = G_UNDECIDED; g.inc = true; return latch(); }
    Problem pb;
    pb.key = keys;
    pb.d.resize(K);
    bool nz = false;
    for (int32_t j = 0; j < K; ++j) {
        pb.d[j] = u.kv[j].second - (l ? l->kv[j].second : 0) - g.own[j];
        nz |= pb.d[j] != 0;
    }
    for (int32_t j = 0; j < K; ++j)
        if (pb.d[j] < 0) { code = JTB_TP_KEY; key = keys[j]; delta = pb.d[j]; return latch(); }
    if (!nz) return latch();
    const int32_t ivl = l ? l->inv : -1;
    auto take = [&](int32_t t) {
        const XTransfer& x = S.T[t];
        if (x.fate == JTB_T_FAIL || !(x.inv < u.comp) || !(x.A < u.comp) || x.M < ivl || x.amount <= 0) return true;
        if (round > 0 && !(W[t].win && W[t].lo <= i && i <= W[t].hi && owner[t] < 0)) return true;
        const int32_t jd = W[t].jd, jc = W[t].jc;
        if (jd < 0 && jc < 0) return true;
        if ((jd >= 0 && x.amount > pb.d[jd]) || (jc >= 0 && x.amount > pb.d[jc])) return true;
        pb.P.push_back({x.id, x.amount, jd, jc, t});
        return pb.P.size() <= (size_t)JTB_TP_MAX_GATHER;
    };
    bool fits = true;
    for (int64_t j = std::lower_bound(X.ok_inv.begin(), X.ok_inv.end(), u.comp) - X.ok_inv.begin() - 1;
         fits && j >= 0 && X.ok_pmax[j] >= ivl; --j)
        fits = take(X.ok[j]);
    for (int32_t c = 0; c < K && fits; ++c) {
        if (pb.d[c] <= 0) continue;
        const int64_t bc = std::lower_bound(X.crashed_inv[c].begin(), X.crashed_inv[c].end(), u.comp) -
                           X.crashed_inv[c].begin();
        for (int64_t j = 0; j < bc && fits; ++j) fits = take(X.crashed[c][j]);
    }
    if (!fits) { code = G_UNDECIDED; g.inc = true; return latch(); }
    Search s(pb, -1, max_nodes);
    int32_t root_key;
    std::vector<int32_t> forced;
    std::vector<uint8_t> st;
    const Verdict v = s.run(root_key, g.kept, &forced, &st);
    nodes += s.nodes;
    for (size_t c = 0; c < pb.P.size(); ++c)
        if (st[c] != OUT) g.poss.push_back(pb.P[c].t);
    for (int32_t c : forced) g.forced.push_back(pb.P[c].t);
    if (v == EXPLAINED) return latch();
    if (v == UNDECIDED) { code = G_UNDECIDED; return latch(); }
    code = JTB_TP_JOINT;
    key = root_key;
    for (int32_t k = 0; k < K; ++k) {
        Search sk(pb, k, max_nodes);
        int32_t rk, kp;
        const Verdict vk = sk.run(rk, kp);
        nodes += sk.nodes;
        if (vk == UNEXPLAINED) { code = JTB_TP_KEY; key = keys[k]; delta = pb.d[k]; break; }
    }
    latch();
}

}  // namespace

extern "C" {

const char* jtbm_tp_last_error(void) { return g_err.c_str(); }

int jtbm_check_transfer_placement(const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t flags,
                                  int32_t algo, jtb_tp_shard* shards, jtb_tp_result* out) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (max_nodes <= 0) max_nodes = JTB_TP_DEFAULT_MAX_NODES;
    if (max_rounds <= 0) max_rounds = JTB_TP_DEFAULT_MAX_ROUNDS;
    memset(out, 0, sizeof *out);
    int64_t n_records = 0, n_reads = 0;
    std::vector<jtb_tp_shard> tmp(h->n_shards);
    try {
        for (int32_t s = 0; s < h->n_shards; ++s) {
            Shard S;
            if (int rc = parse_shard(h, s, S, n_records)) return rc;
            n_reads += (int64_t)S.R.size();
            if (n_reads > INT_MAX) { g_err = "more than 2^31-1 reads"; return -2; }
            classify_inputs(S);
            jtb_tp_shard& o = tmp[s];
            memset(&o, 0, sizeof o);
            o.valid = JTB_VALID;
            o.n_reads = (int32_t)S.R.size();
            o.n_transfers = (int32_t)S.T.size();
            o.witness_index = o.lower_index = o.key = o.other_index = o.round = -1;
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
                continue;
            }
            if (S.R.empty()) continue;
            std::vector<int32_t> ord(S.R.size());
            std::vector<__int128> sum(S.R.size(), 0);
            for (size_t r = 0; r < S.R.size(); ++r) {
                ord[r] = (int32_t)r;
                for (auto& kv : S.R[r].kv) sum[r] += kv.second;
            }
            std::stable_sort(ord.begin(), ord.end(), [&](int32_t a, int32_t b) {
                return sum[a] != sum[b] ? sum[a] < sum[b] : S.R[a].inv < S.R[b].inv;
            });
            const int32_t n = (int32_t)ord.size(), K = (int32_t)keys.size(), nT = (int32_t)S.T.size();
            const std::vector<Window> W = windows(S, keys, ord);
            auto upper = [&](int32_t i) -> const XRead& { return S.R[ord[i]]; };
            auto lower = [&](int32_t i) { return i > 0 ? &S.R[ord[i - 1]] : nullptr; };
            if (algo == TP_BRUTE) {
                Brute b{S, W, std::vector<std::vector<int64_t>>(n, std::vector<int64_t>(K)), {}};
                bool neg = false;
                for (int32_t i = 0; i < n; ++i)
                    for (int32_t k = 0; k < K; ++k)
                        neg |= (b.need[i][k] = upper(i).kv[k].second - (lower(i) ? lower(i)->kv[k].second : 0)) < 0;
                for (int32_t t = 0; t < nT; ++t)
                    if (W[t].win) b.ts.push_back(t);
                o.valid = !neg && b.go(0) ? JTB_VALID : JTB_INVALID;
                continue;
            }
            const Index X(S, keys);
            std::vector<Gap> G(n);
            for (auto& g : G) g.own.assign(K, 0);
            std::vector<int32_t> owner(nT, -1), dround(nT, -1), dg1(nT), dg2(nT), lround(nT, -1);
            std::vector<char> run(n, 1);
            int32_t round = 0;
            for (;; ++round) {
                for (int32_t i = 0; i < n; ++i)
                    if (run[i]) run_gap(S, keys, X, W, owner, upper(i), lower(i), i, round, max_nodes, o.nodes, G[i]);
                o.rounds = round + 1;
                // the owner, PLACE and LOST pass over this round's state
                std::vector<std::vector<int32_t>> forced(nT), poss(nT);
                for (int32_t i = 0; i < n; ++i) {
                    if (run[i])
                        for (int32_t t : G[i].forced) forced[t].push_back(i);
                    for (int32_t t : G[i].poss)
                        if (W[t].lo <= i && i <= W[t].hi) poss[t].push_back(i);
                }
                std::vector<int32_t> inc(n + 1, 0);
                for (int32_t i = 0; i < n; ++i) inc[i + 1] = inc[i] + G[i].inc;
                std::vector<int32_t> dirty(n + 1, 0);
                bool changed = false;
                for (int32_t t = 0; t < nT; ++t) {
                    if (!W[t].win || owner[t] >= 0 || dround[t] >= 0 || lround[t] >= 0) continue;
                    int32_t g = -1;
                    if (forced[t].size() >= 2) {
                        std::sort(forced[t].begin(), forced[t].end());
                        dround[t] = round;
                        dg1[t] = forced[t][0];
                        dg2[t] = forced[t][1];
                    } else if (forced[t].size() == 1) {
                        g = forced[t][0];
                    } else if (W[t].must && (W[t].lo > W[t].hi || inc[W[t].hi + 1] == inc[W[t].lo])) {
                        if (poss[t].empty()) lround[t] = round;
                        else if (poss[t].size() == 1) g = poss[t][0];
                    }
                    if (g < 0) continue;
                    owner[t] = g;
                    changed = true;
                    if (W[t].jd >= 0) G[g].own[W[t].jd] += S.T[t].amount;
                    if (W[t].jc >= 0) G[g].own[W[t].jc] += S.T[t].amount;
                    if (W[t].lo <= W[t].hi) { dirty[W[t].lo]++; dirty[W[t].hi + 1]--; }
                }
                if (round + 1 >= max_rounds || (round >= 1 && !changed)) break;
                for (int32_t i = 0, d = 0; i < n; ++i) {
                    d += dirty[i];
                    run[i] = round == 0 || d > 0;
                }
            }
            // counts, verdict and witness
            uint64_t wbest = ~0ull;
            int64_t wid = 0;
            int32_t wt = -1;
            for (int32_t i = 0; i < n; ++i) {
                const Gap& g = G[i];
                if (g.lcode) {
                    o.count_by_kind[g.lcode - 1]++;
                    wbest = std::min(wbest, (uint64_t)i << 3 | (uint64_t)g.lcode);
                } else if (g.code == G_EXPLAINED) {
                    o.n_explained++;
                } else {
                    o.n_undecided++;
                }
            }
            for (int32_t t = 0; t < nT; ++t) {
                o.n_placed += owner[t] >= 0;
                uint64_t k = ~0ull;
                if (dround[t] >= 0) { o.count_by_kind[2]++; k = (uint64_t)dg2[t] << 3 | JTB_TP_DOUBLE; }
                if (lround[t] >= 0) { o.count_by_kind[3]++; k = (uint64_t)W[t].hi << 3 | JTB_TP_LOST; }
                if (k < wbest || (k == wbest && wt >= 0 && S.T[t].id < wid)) { wbest = k; wt = t; wid = S.T[t].id; }
            }
            if (wbest == ~0ull) {
                o.valid = o.n_undecided ? JTB_UNKNOWN : JTB_VALID;
                continue;
            }
            const int32_t wg = (int32_t)(wbest >> 3);
            o.valid = JTB_INVALID;
            o.kind = (int32_t)(wbest & 7);
            o.witness_index = upper(wg).comp_index;
            o.lower_index = wg > 0 ? S.R[ord[wg - 1]].comp_index : -1;
            o.n_eligible = G[wg].kept;
            if (o.kind == JTB_TP_DOUBLE) {
                o.transfer_id = S.T[wt].id;
                o.other_index = upper(dg1[wt]).comp_index;
                o.round = dround[wt];
            } else if (o.kind == JTB_TP_LOST) {
                o.transfer_id = S.T[wt].id;
                o.other_index = h->index[h->shard_off[s] + S.T[wt].M];
                o.round = lround[wt];
            } else {
                o.key = G[wg].lkey;
                o.delta = o.kind == JTB_TP_KEY ? G[wg].ldelta : 0;
                o.round = G[wg].lround;
            }
        }
    } catch (int) {
        return -2;
    }
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const jtb_tp_shard& o = shards[s] = tmp[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_explained += o.n_explained;
        out->n_unexplained += o.count_by_kind[0] + o.count_by_kind[1];
        out->n_double += o.count_by_kind[2];
        out->n_lost += o.count_by_kind[3];
        out->n_undecided += o.n_undecided;
        out->n_placed += o.n_placed;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
