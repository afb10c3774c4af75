// repaired_witness.cpp — CPU oracle of the repaired serial witness (TEST INFRASTRUCTURE ONLY; the library never calls
// it).
//
// RW_SEARCH is the library's decision, shard by shard: SW_SEARCH's TP_SEARCH and witness (the Witness of
// witness_common.h); a shard it proves is returned as SW_SEARCH returns it.  On NO_WITNESS or REAL_TIME, up to
// max_repairs repair rounds: the blame of the failure as (gap, transfer) bans, the release of the blamed gaps and the
// failing one, the witness rounds again with banned pairs and transfers that complete by P^_g (the point of g's lower
// read from the reads and the owned transfers, recomputed every round) out of the gather, then the unchanged re-sum
// and real-time pass.  Node counts, rounds, repairs and bans are the library's.  The loop is repair_common.h's, with
// no lift steps.
#include "repair_common.h"

namespace {

constexpr int RW_SEARCH = 1;

void roll_rw(jtb_rw_result*, const jtb_rw_shard&) {}

}  // namespace

extern "C" {

const char* jtbm_rw_last_error(void) { return g_err.c_str(); }

int jtbm_check_repaired_witness(const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t max_repairs,
                                int32_t flags, int32_t algo, int32_t* commit_read, jtb_rw_shard* shards,
                                jtb_rw_result* out) {
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (algo != RW_SEARCH) { g_err = "unknown algorithm"; return -2; }
    return repaired_check(h, max_nodes, max_rounds, max_repairs, 0, commit_read, shards, out, roll_rw);
}

}  // extern "C"
