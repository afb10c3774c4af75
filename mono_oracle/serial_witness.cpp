// serial_witness.cpp — CPU oracle of the serial-witness check (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// SW_SEARCH is the library's decision, shard by shard: TP_SEARCH (tp_search in gaps_common.h, as the transfer-placement
// oracle runs it); for a shard it calls VALID, the witness rounds (every unfixed gap gathers as a TP_SEARCH round >= 1
// does and keeps the search's first solution; a gap is fixed when no smaller gap of the round chose one of its
// transfers), D_g = owned + fixed, the greedy real-time pass over the reads in the gap order, the re-sum of every
// gap's counters, and commit_read (the Witness of witness_common.h, run once).  Node counts and rounds are the
// library's.
#include <chrono>
#include <cstring>

#include "witness_common.h"

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
    Witness x(S, keys, ord, T);
    int32_t rounds = 0;
    const int32_t failed = x.rounds(max_nodes, max_rounds, {}, {}, rounds, o.nodes);
    o.rounds = rounds;
    if (failed >= 0) {
        o.valid = JTB_UNKNOWN;
        o.cause = JTB_CAUSE_NO_WITNESS;
        o.fail_index = x.upper(failed).comp_index;
        return 0;
    }
    if (!x.check()) {
        g_err = "the counters of a serial witness do not add up";
        return -1;
    }
    x.verdict(o, w.commit);
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
