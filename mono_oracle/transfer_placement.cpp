// transfer_placement.cpp — CPU oracle of the transfer-placement check (TEST INFRASTRUCTURE ONLY; the library never
// calls it).
//
// Both deciders parse a shard, order its reads and form its gaps as the read-gap oracle does (gaps_common.h), give
// every transfer its window of gaps [lo, hi] and fill jtb_tp_shard as jtb_check_transfer_placement does.
// TP_BRUTE is the definition: every assignment of each windowed transfer to one gap of its window, or to none for a
// may transfer, and whether some assignment makes every gap sum to Delta on every key.  No caps; tiny histories only.
// TP_SEARCH is the library's (tp_search in gaps_common.h, which the serial-witness oracle runs too): round 0 is
// RG_SEARCH gap for gap, then the owner / PLACE / LOST pass after every round, the re-runs of round 1 (every gap) and
// of the dirtied gaps after it with Delta' and the in-window gather, the latch and the witness.  Node counts and rounds
// are the library's.
#include <chrono>
#include <cstring>
#include <memory>

#include "gaps_common.h"

namespace {

constexpr int TP_BRUTE = 0, TP_SEARCH = 1;

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
            std::vector<int32_t> keys, ord;
            bool partial;
            shard_order(S, keys, partial, ord);
            if (partial) {
                o.valid = JTB_UNKNOWN;
                o.cause = JTB_CAUSE_PARTIAL_READ;
                continue;
            }
            if (S.R.empty()) continue;
            const int32_t n = (int32_t)ord.size(), K = (int32_t)keys.size(), nT = (int32_t)S.T.size();
            if (algo == TP_BRUTE) {
                const std::vector<Window> W = windows(S, keys, ord);
                auto upper = [&](int32_t i) -> const XRead& { return S.R[ord[i]]; };
                auto lower = [&](int32_t i) { return i > 0 ? &S.R[ord[i - 1]] : nullptr; };
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
            TpState T;
            tp_search(h, s, S, keys, ord, max_nodes, max_rounds, o, T);
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
