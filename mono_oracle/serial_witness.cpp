// serial_witness.cpp — CPU oracle of the serial-witness check (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// SW_SEARCH is the library's decision, shard by shard: TP_SEARCH (tp_search in gaps_common.h, as the transfer-placement
// oracle runs it); for a shard it calls VALID, the witness rounds (every unfixed gap gathers as a TP_SEARCH round >= 1
// does and keeps the search's first solution; a gap is fixed when no smaller gap of the round chose one of its
// transfers), D_g = owned + fixed, the greedy real-time pass over the reads in the gap order, the re-sum of every
// gap's counters, and commit_read.  Node counts and rounds are the library's.
#include <chrono>
#include <cstring>

#include "gaps_common.h"

namespace {

constexpr int SW_SEARCH = 1;

struct SwOut {
    jtb_sw_shard o;
    std::vector<int32_t> commit;   // per transfer of the shard
};

// the witness, real time and commit_read of a shard TP_SEARCH called VALID
int witness(const Shard& S, const std::vector<int32_t>& keys, const std::vector<int32_t>& ord, TpState& T,
            int64_t max_nodes, int32_t max_rounds, SwOut& w) {
    jtb_sw_shard& o = w.o;
    const int32_t n = (int32_t)ord.size(), K = (int32_t)keys.size(), nT = (int32_t)S.T.size();
    const std::vector<Window>& W = T.W;
    std::vector<int32_t>& owner = T.owner;
    auto upper = [&](int32_t i) -> const XRead& { return S.R[ord[i]]; };
    auto lower = [&](int32_t i) { return i > 0 ? &S.R[ord[i - 1]] : nullptr; };
    auto delta = [&](int32_t i, int32_t j) {
        return upper(i).kv[j].second - (lower(i) ? lower(i)->kv[j].second : 0) - T.G[i].own[j];
    };
    const Index X(S, keys);
    std::vector<char> fixed(n, 1);
    for (int32_t i = 0; i < n; ++i)
        for (int32_t j = 0; j < K; ++j) fixed[i] &= delta(i, j) == 0;
    // the witness rounds
    std::vector<std::vector<int32_t>> chosen(n);
    for (int32_t round = 0;; ++round) {
        int32_t first = -1;
        for (int32_t i = 0; i < n && first < 0; ++i)
            if (!fixed[i]) first = i;
        if (first < 0) break;
        if (round >= max_rounds) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_NO_WITNESS;
            o.fail_index = upper(first).comp_index;
            return 0;
        }
        o.rounds = round + 1;
        int32_t failed = -1;
        for (int32_t i = 0; i < n; ++i) {
            if (fixed[i]) continue;
            chosen[i].clear();
            Problem pb;
            pb.key = keys;
            pb.d.resize(K);
            bool neg = false;
            for (int32_t j = 0; j < K; ++j) neg |= (pb.d[j] = delta(i, j)) < 0;
            bool ok = !neg && gather_gap(S, X, W, owner, upper(i), lower(i), i, 1, pb);
            if (ok) {
                Search s(pb, -1, max_nodes);
                int32_t root_key, kept;
                std::vector<uint8_t> sol;
                ok = s.run(root_key, kept, nullptr, nullptr, &sol) == EXPLAINED;
                o.nodes += s.nodes;
                if (ok)
                    for (size_t c = 0; c < pb.P.size(); ++c)
                        if (sol[c] == IN) chosen[i].push_back(pb.P[c].t);
            }
            if (!ok && failed < 0) failed = i;
        }
        if (failed >= 0) {
            o.valid = JTB_UNKNOWN;
            o.cause = JTB_CAUSE_NO_WITNESS;
            o.fail_index = upper(failed).comp_index;
            return 0;
        }
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
                for (int32_t t : chosen[i]) owner[t] = i;
            }
    }
    // the counters of every gap from D_g
    std::vector<std::vector<int64_t>> sum(n, std::vector<int64_t>(K, 0));
    for (int32_t t = 0; t < nT; ++t) {
        if (owner[t] < 0) continue;
        if (W[t].jd >= 0) sum[owner[t]][W[t].jd] += S.T[t].amount;
        if (W[t].jc >= 0) sum[owner[t]][W[t].jc] += S.T[t].amount;
    }
    for (int32_t i = 0; i < n; ++i)
        for (int32_t j = 0; j < K; ++j)
            if (sum[i][j] != upper(i).kv[j].second - (lower(i) ? lower(i)->kv[j].second : 0)) {
                g_err = "the counters of a serial witness do not add up";
                return -1;
            }
    // real time: Q[i] = P_{i+1}, the point of the read at position i
    std::vector<int32_t> gmax(n, INT_MIN), gmin(n, INT_MAX);
    for (int32_t t = 0; t < nT; ++t) {
        if (owner[t] < 0) continue;
        gmax[owner[t]] = std::max(gmax[owner[t]], S.T[t].inv);
        gmin[owner[t]] = std::min(gmin[owner[t]], S.T[t].okcomp);
    }
    std::vector<int32_t> Q(n);
    uint64_t best = ~0ull;
    for (int32_t i = 0; i < n; ++i) {
        Q[i] = std::max({i > 0 ? Q[i - 1] : INT_MIN, upper(i).inv, gmax[i]});
        if (i > 0 && gmin[i] <= Q[i - 1]) best = std::min(best, (uint64_t)i << 1);
        if (Q[i] >= upper(i).comp) best = std::min(best, (uint64_t)i << 1 | 1);
    }
    for (int32_t t = 0; t < nT; ++t)
        if (S.T[t].fate == JTB_T_OK && W[t].win && owner[t] < 0 && S.T[t].okcomp <= Q[n - 1])
            best = std::min(best, (uint64_t)n << 1);
    if (best != ~0ull) {
        o.valid = JTB_UNKNOWN;
        o.cause = JTB_CAUSE_REAL_TIME;
        const int32_t at = (int32_t)(best >> 1);
        if (best & 1) {
            o.fail_index = upper(at).comp_index;
            return 0;
        }
        int32_t wt = -1;
        for (int32_t t = 0; t < nT; ++t) {
            const bool fails = at < n ? owner[t] == at && S.T[t].okcomp <= Q[at - 1]
                                      : S.T[t].fate == JTB_T_OK && W[t].win && owner[t] < 0 &&
                                            S.T[t].okcomp <= Q[n - 1];
            if (fails && (wt < 0 || S.T[t].id < S.T[wt].id)) wt = t;
        }
        o.fail_index = S.T[wt].cidx;
        o.transfer_id = S.T[wt].id;
        return 0;
    }
    for (int32_t t = 0; t < nT; ++t) {
        const XTransfer& x = S.T[t];
        if (owner[t] >= 0) {
            w.commit[t] = upper(owner[t]).comp_index;
            o.n_committed++;
            o.n_committed_crashed += x.fate != JTB_T_OK;
        } else if (x.fate == JTB_T_OK && W[t].win) {
            w.commit[t] = JTB_SW_AFTER;
            o.n_after++;
        } else if (x.fate == JTB_T_OK) {
            w.commit[t] = JTB_SW_FREE;
        }
    }
    return 0;
}

}  // namespace

extern "C" {

const char* jtbm_sw_last_error(void) { return g_err.c_str(); }

int jtbm_check_serial_witness(const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t flags, int32_t algo,
                              int32_t* commit_read, jtb_sw_shard* shards, jtb_sw_result* out) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (algo != SW_SEARCH) { g_err = "unknown algorithm"; return -2; }
    if (max_nodes <= 0) max_nodes = JTB_TP_DEFAULT_MAX_NODES;
    if (max_rounds <= 0) max_rounds = JTB_TP_DEFAULT_MAX_ROUNDS;
    memset(out, 0, sizeof *out);
    int64_t n_records = 0, n_reads = 0;
    std::vector<SwOut> tmp(h->n_shards);
    try {
        for (int32_t s = 0; s < h->n_shards; ++s) {
            Shard S;
            if (int rc = parse_shard(h, s, S, n_records)) return rc;
            n_reads += (int64_t)S.R.size();
            if (n_reads > INT_MAX) { g_err = "more than 2^31-1 reads"; return -2; }
            classify_inputs(S);
            SwOut& w = tmp[s];
            jtb_sw_shard& o = w.o;
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
            if (S.R.empty()) {   // no read observes a counter: every :ok transfer commits freely
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
                continue;
            }
            if (int rc = witness(S, keys, ord, T, max_nodes, max_rounds, w)) return rc;
            if (o.valid != JTB_VALID) {
                o.n_committed = o.n_committed_crashed = o.n_after = 0;
                std::fill(w.commit.begin(), w.commit.end(), JTB_SW_NEVER);
            }
        }
    } catch (int) {
        return -2;
    }
    int64_t at = 0;
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const jtb_sw_shard& o = shards[s] = tmp[s].o;
        if (commit_read) std::copy(tmp[s].commit.begin(), tmp[s].commit.end(), commit_read + at);
        at += (int64_t)tmp[s].commit.size();
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_committed += o.n_committed;
        out->n_committed_crashed += o.n_committed_crashed;
        out->n_after += o.n_after;
        out->nodes += o.nodes;
        out->rounds = std::max(out->rounds, (int64_t)o.rounds);
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
