// lifted_witness.cpp — CPU oracle of the lifted serial witness (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// LW_SEARCH is the library's decision, shard by shard: RW_SEARCH's witness and repairs, and where a NO_WITNESS repair
// records no new ban, a lift step in place of the stop (repair_common.h): the failing gaps steal again with their own
// bans ignored (a pair lifted before and banned again stays banned) and P^0 (the reads' invocations alone) in place of
// P^; the bans a kept thief's loot hits in the thief are lifted, the chosen transfers it takes banned in their gaps,
// and the repairs resume.  At most max_lifts lift steps and max_repairs + max_lifts repairs per shard; a lift step
// that lifts nothing ends the shard.  Node counts, rounds, repairs, bans and lifts are the library's.
#include "repair_common.h"

namespace {

constexpr int LW_SEARCH = 1;

void roll_lw(jtb_lw_result* out, const jtb_lw_shard& o) {
    out->lifts = std::max(out->lifts, (int64_t)o.lifts);
    out->n_lifted += o.n_lifted;
}

}  // namespace

extern "C" {

const char* jtbm_lw_last_error(void) { return g_err.c_str(); }

int jtbm_check_lifted_witness(const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t max_repairs,
                              int32_t max_lifts, int32_t flags, int32_t algo, int32_t* commit_read,
                              jtb_lw_shard* shards, jtb_lw_result* out) {
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (algo != LW_SEARCH) { g_err = "unknown algorithm"; return -2; }
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    return repaired_check(h, max_nodes, max_rounds, max_repairs, max_lifts, commit_read, shards, out, roll_lw);
}

}  // extern "C"
