// read_gaps.cpp — CPU oracle of the read-gap check (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// Both deciders parse a shard the way the read-explanation oracle does (reads and lookups paired with the latest invoke
// of their process, every [:t ...] micro-op a transfer paired with the next event of its process, M(t) and A(t) from
// the lookups), order the :ok reads of a full-key shard by (S as 128 bits, invocation position), stably over completion
// order, and decide every gap between successive reads; they fill jtb_rg_shard as jtb_check_read_gaps does.
// RG_BRUTE is the definition: every subset of a gap's eligible transfers that fit under Delta (no member of a solution
// exceeds Delta_k on a key; the kinds are defined over these), no caps (tiny histories only); a transfer in every
// solution of two gaps is DOUBLE.
// RG_SEARCH is the library's decision: the amount filter while gathering, the same caps, the root pruning fixpoint in
// Jacobi rounds, at most 64 free candidates in the canonical order (amount descending, then id), a depth-first search
// including before excluding, the same fixpoint at every node and the node budget; a transfer the root pruning forces
// into two gaps is DOUBLE.  Node counts are the library's.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../include/jtb_check.h"

namespace {

constexpr int RG_BRUTE = 0, RG_SEARCH = 1;
constexpr int32_t NONE = INT_MAX;
// per-gap codes of the optional per-gap output
constexpr int8_t G_EXPLAINED = 0, G_UNDECIDED = 3;

thread_local std::string g_err;

struct XRead {
    int32_t inv, comp, comp_index;
    std::vector<std::pair<int32_t, int64_t>> kv;   // sorted by key
};

struct XTransfer {
    int64_t id;
    int32_t debit, credit, amount, inv;
    int32_t fate = -1, okcomp = NONE;
    int32_t M = NONE, A = -1;
};

struct XLookup {
    int32_t inv, comp;
    std::unordered_set<int64_t> ids;
};

struct Shard {
    std::vector<XRead> R;
    std::vector<XTransfer> T;
    std::vector<XLookup> L;
};

inline int64_t rec_id(const int32_t* r) { return (int64_t)(((uint64_t)(uint32_t)r[1] << 32) | (uint32_t)r[0]); }

int fail(const char* fmt, int32_t index, int64_t x = 0) {
    char buf[256];
    snprintf(buf, sizeof buf, fmt, index, (long long)x);
    g_err = buf;
    return -2;
}

int parse_shard(const jtb_history* h, int32_t s, Shard& S, int64_t& n_records) {
    const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
    std::unordered_map<int32_t, int32_t> last_inv;
    std::unordered_map<int32_t, std::vector<size_t>> open;
    std::unordered_set<int64_t> ids;
    for (int64_t e = lo; e < hi; ++e) {
        const int32_t p = h->process[e], pos = (int32_t)(e - lo);
        if (p < 0) continue;
        auto ot = open.find(p);
        if (ot != open.end()) {
            if (h->type[e] != JTB_T_INVOKE)
                for (size_t t : ot->second) {
                    S.T[t].fate = h->type[e];
                    if (h->type[e] == JTB_T_OK) S.T[t].okcomp = pos;
                }
            open.erase(ot);
        }
        const int32_t len = h->payload_len[e];
        const int64_t off = h->payload_off[e];
        if (h->type[e] == JTB_T_INVOKE) {
            last_inv[p] = pos;
            if (h->f[e] != JTB_F_TRANSFER) continue;
            if (len <= 0) return fail("transfer at :index %d: an invoke without ids", h->index[e]);
            if (len % 5 != 0) return fail("transfer at :index %d: payload length %lld is not a multiple of 5",
                                          h->index[e], len);
            if (off < 0 || off + len > h->n_payload) return fail("transfer at :index %d: payload out of range",
                                                                h->index[e]);
            auto& o = open[p];
            for (int32_t j = 0; j < len; j += 5) {
                const int32_t* r = h->payload + off + j;
                if (r[4] < 0) return fail("transfer at :index %d: negative amount %lld", h->index[e], r[4]);
                if (r[2] < 0 || r[2] >= (1 << 30) || r[3] < 0 || r[3] >= (1 << 30))
                    return fail("transfer at :index %d: account outside [0, 2^30)", h->index[e]);
                const int64_t id = rec_id(r);
                if (!ids.insert(id).second)
                    return fail("transfer at :index %d: id %lld is carried by two transfer invokes", h->index[e], id);
                XTransfer t;
                t.id = id; t.debit = r[2]; t.credit = r[3]; t.amount = r[4]; t.inv = pos;
                o.push_back(S.T.size());
                S.T.push_back(t);
            }
            continue;
        }
        if (h->type[e] != JTB_T_OK || len < 0) continue;
        auto it = last_inv.find(p);
        const int32_t inv = it == last_inv.end() ? -1 : it->second;
        if (h->f[e] == JTB_F_LOOKUP) {
            if (len % 5 != 0) return fail("lookup at :index %d: payload length %lld is not a multiple of 5",
                                          h->index[e], len);
            if (off < 0 || off + len > h->n_payload) return fail("lookup at :index %d: payload out of range",
                                                                h->index[e]);
            n_records += len / 5;
            if (n_records > INT_MAX) { g_err = "more than 2^31-1 lookup records"; return -2; }
            XLookup l{inv, pos, {}};
            for (int32_t j = 0; j < len; j += 5) l.ids.insert(rec_id(h->payload + off + j));
            S.L.push_back(std::move(l));
            continue;
        }
        if (h->f[e] != JTB_F_READ) continue;
        if (len % 3 != 0 || off < 0 || off + len > h->n_payload)
            return fail("read at :index %d: malformed payload", h->index[e]);
        XRead r{inv, pos, h->index[e], {}};
        for (int32_t j = 0; j < len; j += 3) {
            const int32_t* t = h->payload + off + j;
            r.kv.push_back({t[0], (int64_t)(((uint64_t)(uint32_t)t[2] << 32) | (uint32_t)t[1])});
        }
        std::sort(r.kv.begin(), r.kv.end());
        for (size_t j = 1; j < r.kv.size(); ++j)
            if (r.kv[j].first == r.kv[j - 1].first)
                return fail("read at :index %d observes key %lld twice", h->index[e], r.kv[j].first);
        S.R.push_back(std::move(r));
    }
    return 0;
}

// M(t) = min(:ok completion, earliest completion of an :ok lookup returning t); A(t) = latest invocation of an :ok
// lookup (with an invocation) lacking t
void classify_inputs(Shard& S) {
    for (auto& t : S.T) {
        t.M = t.okcomp;
        for (auto& l : S.L) {
            if (l.ids.count(t.id)) t.M = std::min(t.M, l.comp);
            else if (l.inv >= 0) t.A = std::max(t.A, l.inv);
        }
    }
}

struct Cand {
    int64_t id;
    int32_t a, jd, jc;   // jd / jc: column of the debit / credit key, -1 unobserved
    int32_t t;           // the transfer
};

// One gap's subset-sum problem: candidates and Delta per column.
struct Problem {
    std::vector<Cand> P;
    std::vector<int64_t> d;
    std::vector<int32_t> key;
};

// ---- RG_BRUTE ----------------------------------------------------------------------------------------------------
// the solutions of P with sum d on every key (only >= 0: on that key alone); first: stop at the first one.  Returns
// whether one exists; all = the AND of the solutions' masks
bool brute(const Problem& pb, int32_t only, bool first, uint64_t& all) {
    const size_t n = pb.P.size(), K = pb.d.size();
    if (n > 24) { g_err = "RG_BRUTE: more than 24 candidates"; throw 1; }
    std::vector<int64_t> s(K);
    bool any = false;
    all = ~0ull;
    for (uint64_t x = 0; x < (1ull << n); ++x) {
        std::fill(s.begin(), s.end(), 0);
        for (size_t c = 0; c < n; ++c)
            if (x >> c & 1) {
                if (pb.P[c].jd >= 0) s[pb.P[c].jd] += pb.P[c].a;
                if (pb.P[c].jc >= 0) s[pb.P[c].jc] += pb.P[c].a;
            }
        bool ok = true;
        for (size_t k = 0; k < K && ok; ++k)
            if (only < 0 || (int32_t)k == only) ok = s[k] == pb.d[k];
        if (!ok) continue;
        any = true;
        all &= x;
        if (first) return true;
    }
    return any;
}

// ---- RG_SEARCH (K10's search) ------------------------------------------------------------------------------------
enum { UND = 0, IN = 1, OUT = 2 };
enum Verdict { EXPLAINED, UNEXPLAINED, UNDECIDED };

struct Search {
    const Problem& pb;
    int32_t only;
    int64_t max_nodes, nodes = 0;
    std::vector<int64_t> ins, av;

    Search(const Problem& p, int32_t o, int64_t mx) : pb(p), only(o), max_nodes(mx), ins(p.d.size()), av(p.d.size()) {}

    int32_t rel(int32_t j) const { return only < 0 || j == only ? j : -1; }

    bool prune(const std::vector<int32_t>& ids, std::vector<uint8_t>& st, const std::vector<int64_t>& base,
               int32_t& bad) {
        const int32_t K = (int32_t)base.size();
        for (;;) {
            std::fill(ins.begin(), ins.end(), 0);
            std::fill(av.begin(), av.end(), 0);
            for (int32_t c : ids) {
                if (st[c] == OUT) continue;
                auto& v = st[c] == IN ? ins : av;
                const int32_t kd = rel(pb.P[c].jd), kc = rel(pb.P[c].jc);
                if (kd >= 0) v[kd] += pb.P[c].a;
                if (kc >= 0) v[kc] += pb.P[c].a;
            }
            bad = -1;
            for (int32_t k = 0; k < K && bad < 0; ++k) {
                if (rel(k) < 0) continue;
                const int64_t need = base[k] - ins[k];
                if (need < 0 || need > av[k]) bad = k;
            }
            if (bad >= 0) return false;
            std::vector<std::pair<int32_t, uint8_t>> upd;
            for (int32_t c : ids) {
                if (st[c] != UND) continue;
                const int32_t ks[2] = {rel(pb.P[c].jd), rel(pb.P[c].jc)};
                const int64_t a = pb.P[c].a;
                bool drop = false, force = false;
                for (int32_t k : ks)
                    if (k >= 0 && a > base[k] - ins[k]) drop = true;
                for (int32_t k : ks)
                    if (!drop && k >= 0 && av[k] - a < base[k] - ins[k]) force = true;
                if (drop) upd.push_back({c, OUT});
                else if (force) upd.push_back({c, IN});
            }
            if (upd.empty()) return true;
            for (auto& [c, v] : upd) st[c] = v;
        }
    }

    bool dfs(const std::vector<int32_t>& F, std::vector<uint8_t>& st, const std::vector<int64_t>& base) {
        int32_t b = -1;
        for (int32_t c : F)
            if (st[c] == UND) { b = c; break; }
        for (uint8_t v : {(uint8_t)IN, (uint8_t)OUT}) {
            if (++nodes > max_nodes) throw 2;
            std::vector<uint8_t> s2 = st;
            s2[b] = v;
            int32_t bad;
            if (!prune(F, s2, base, bad)) continue;
            bool any = false;
            for (int32_t c : F) any |= s2[c] == UND;
            if (!any || dfs(F, s2, base)) return true;
        }
        return false;
    }

    // root_key: the smallest key the root pruning found unreachable, -1; kept: candidates the root did not drop;
    // forced: the candidates a feasible root pruning forces in
    Verdict run(int32_t& root_key, int32_t& kept, std::vector<int32_t>* forced = nullptr) {
        const int32_t n = (int32_t)pb.P.size();
        std::vector<uint8_t> st(n, UND);
        std::vector<int32_t> all(n);
        for (int32_t c = 0; c < n; ++c) {
            all[c] = c;
            if (rel(pb.P[c].jd) < 0 && rel(pb.P[c].jc) < 0) st[c] = OUT;
        }
        nodes = 1;
        root_key = -1;
        kept = 0;
        int32_t bad;
        const bool ok = prune(all, st, pb.d, bad);
        for (int32_t c = 0; c < n; ++c) kept += st[c] != OUT;
        if (!ok) { root_key = pb.key[bad]; return UNEXPLAINED; }
        if (forced)
            for (int32_t c = 0; c < n; ++c)
                if (st[c] == IN) forced->push_back(c);
        std::vector<int32_t> F;
        for (int32_t c = 0; c < n; ++c)
            if (st[c] == UND) F.push_back(c);
        if (F.empty()) return EXPLAINED;
        if (F.size() > (size_t)JTB_RG_MAX_FREE) return UNDECIDED;
        std::sort(F.begin(), F.end(), [&](int32_t x, int32_t y) {
            return pb.P[x].a != pb.P[y].a ? pb.P[x].a > pb.P[y].a : pb.P[x].id < pb.P[y].id;
        });
        std::vector<int64_t> base(pb.d.size());
        for (size_t k = 0; k < base.size(); ++k) base[k] = pb.d[k] - ins[k];   // ins: the forced-in of the root
        try {
            return dfs(F, st, base) ? EXPLAINED : UNEXPLAINED;
        } catch (int) {
            return UNDECIDED;
        }
    }
};

struct GapOut {
    int8_t code = G_EXPLAINED;
    int32_t key = -1, n_eligible = 0;
    int64_t delta = 0;
    std::vector<int32_t> forced;   // transfers this gap forces in
};

int32_t col_of(const std::vector<int32_t>& keys, int64_t key) {
    auto it = std::lower_bound(keys.begin(), keys.end(), key, [](int32_t a, int64_t b) { return a < b; });
    return it != keys.end() && *it == key ? (int32_t)(it - keys.begin()) : -1;
}

// RG_SEARCH's sweep structures: the :ok transfers in invocation order (the order of S.T) with the running max of their
// completions, and the crashed (:info, never completed) ones with a positive amount in invocation order, by anchor
// column (the debit key's, else the credit key's; none when the shard observes neither)
struct Index {
    std::vector<int32_t> ok, ok_inv, ok_pmax;
    std::vector<std::vector<int32_t>> crashed, crashed_inv;
    Index(const Shard& S, const std::vector<int32_t>& keys) : crashed(keys.size()), crashed_inv(keys.size()) {
        for (size_t i = 0; i < S.T.size(); ++i) {
            const XTransfer& t = S.T[i];
            if (t.fate == JTB_T_OK) {
                ok.push_back((int32_t)i);
                ok_inv.push_back(t.inv);
                ok_pmax.push_back(std::max(ok_pmax.empty() ? INT_MIN : ok_pmax.back(), t.okcomp));
            } else if (t.fate != JTB_T_FAIL && t.amount > 0) {
                int32_t a = col_of(keys, 2 * (int64_t)t.debit);
                if (a < 0) a = col_of(keys, 2 * (int64_t)t.credit + 1);
                if (a < 0) continue;
                crashed[a].push_back((int32_t)i);
                crashed_inv[a].push_back(t.inv);
            }
        }
    }
};

// one gap: upper read u, lower read l (nullptr for gap 0); X: RG_SEARCH's sweep (nullptr: RG_BRUTE)
GapOut decide_gap(const Shard& S, const std::vector<int32_t>& keys, const Index* X, const XRead& u, const XRead* l,
                  int algo, int64_t max_nodes, int64_t& nodes) {
    GapOut o;
    const int32_t K = (int32_t)keys.size();
    if (algo == RG_SEARCH && K > JTB_RG_MAX_KEYS) { o.code = G_UNDECIDED; return o; }
    Problem pb;
    pb.key = keys;
    pb.d.resize(K);
    bool nz = false;
    for (int32_t j = 0; j < K; ++j) {
        pb.d[j] = u.kv[j].second - (l ? l->kv[j].second : 0);
        if (pb.d[j] < 0) { o.code = JTB_RG_KEY; o.key = keys[j]; o.delta = pb.d[j]; return o; }
        nz |= pb.d[j] != 0;
    }
    if (!nz) return o;
    const int32_t ivl = l ? l->inv : -1;
    auto take = [&](int32_t t) {   // false: more eligible transfers than the gather cap
        const XTransfer& x = S.T[t];
        if (x.fate == JTB_T_FAIL || !(x.inv < u.comp) || !(x.A < u.comp) || x.M < ivl || x.amount <= 0) return true;
        const int32_t jd = col_of(keys, 2 * (int64_t)x.debit), jc = col_of(keys, 2 * (int64_t)x.credit + 1);
        if (jd < 0 && jc < 0) return true;
        if ((jd >= 0 && x.amount > pb.d[jd]) || (jc >= 0 && x.amount > pb.d[jc])) return true;   // fits under Delta
        pb.P.push_back({x.id, x.amount, jd, jc, t});
        return !X || pb.P.size() <= (size_t)JTB_RG_MAX_GATHER;
    };
    bool fits = true;
    if (!X) {
        for (int32_t t = 0; t < (int32_t)S.T.size(); ++t) take(t);
    } else {
        // :ok transfers invoked before u completed, back to the last one whose running max completion is before l's
        // invocation (every earlier one completed before it, so is in l's state); the crashed ones anchored at a key
        // that grew
        for (int64_t j = std::lower_bound(X->ok_inv.begin(), X->ok_inv.end(), u.comp) - X->ok_inv.begin() - 1;
             fits && j >= 0 && X->ok_pmax[j] >= ivl; --j)
            fits = take(X->ok[j]);
        for (int32_t c = 0; c < K && fits; ++c) {
            if (pb.d[c] <= 0) continue;
            const int64_t bc = std::lower_bound(X->crashed_inv[c].begin(), X->crashed_inv[c].end(), u.comp) -
                               X->crashed_inv[c].begin();
            for (int64_t j = 0; j < bc && fits; ++j) fits = take(X->crashed[c][j]);
        }
    }
    if (algo == RG_BRUTE) {
        o.n_eligible = (int32_t)pb.P.size();
        uint64_t all;
        if (brute(pb, -1, false, all)) {
            for (size_t c = 0; c < pb.P.size(); ++c)
                if (all >> c & 1) o.forced.push_back(pb.P[c].t);
            return o;
        }
        o.code = JTB_RG_JOINT;
        for (int32_t k = 0; k < K; ++k)
            if (!brute(pb, k, true, all)) { o.code = JTB_RG_KEY; o.key = keys[k]; o.delta = pb.d[k]; break; }
        return o;
    }
    if (!fits) { o.code = G_UNDECIDED; return o; }
    Search s(pb, -1, max_nodes);
    int32_t root_key, kept;
    std::vector<int32_t> forced;
    const Verdict v = s.run(root_key, kept, &forced);
    nodes += s.nodes;
    o.n_eligible = kept;
    for (int32_t c : forced) o.forced.push_back(pb.P[c].t);
    if (v == EXPLAINED) return o;
    if (v == UNDECIDED) { o.code = G_UNDECIDED; return o; }
    o.code = JTB_RG_JOINT;
    o.key = root_key;
    for (int32_t k = 0; k < K; ++k) {
        Search sk(pb, k, max_nodes);
        int32_t rk, kp;
        const Verdict vk = sk.run(rk, kp);
        nodes += sk.nodes;
        if (vk == UNEXPLAINED) { o.code = JTB_RG_KEY; o.key = keys[k]; o.delta = pb.d[k]; break; }
    }
    return o;
}

}  // namespace

extern "C" {

const char* jtbm_rg_last_error(void) { return g_err.c_str(); }

// per_gap (may be NULL): one code per :ok read in shard-major order, the gaps of a full-key shard in gap order, 3 for
// the reads of a partial-read shard: 0 explained, 1 KEY, 2 JOINT, 3 undecided
int jtbm_check_read_gaps(const jtb_history* h, int64_t max_nodes, int32_t flags, int32_t algo, jtb_rg_shard* shards,
                         jtb_rg_result* out, int8_t* per_gap) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (max_nodes <= 0) max_nodes = JTB_RG_DEFAULT_MAX_NODES;
    memset(out, 0, sizeof *out);
    int64_t n_records = 0, n_reads = 0;
    std::vector<jtb_rg_shard> tmp(h->n_shards);
    std::vector<int8_t> codes;
    try {
        for (int32_t s = 0; s < h->n_shards; ++s) {
            Shard S;
            if (int rc = parse_shard(h, s, S, n_records)) return rc;
            n_reads += (int64_t)S.R.size();
            if (n_reads > INT_MAX) { g_err = "more than 2^31-1 reads"; return -2; }
            classify_inputs(S);
            jtb_rg_shard& o = tmp[s];
            memset(&o, 0, sizeof o);
            o.valid = JTB_VALID;
            o.n_reads = (int32_t)S.R.size();
            o.n_transfers = (int32_t)S.T.size();
            o.witness_index = o.lower_index = o.key = o.other_index = -1;
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
                codes.insert(codes.end(), S.R.size(), G_UNDECIDED);
                continue;
            }
            // the gap order: (S, invocation), stable over completion order
            std::vector<int32_t> ord(S.R.size());
            std::vector<__int128> sum(S.R.size(), 0);
            for (size_t r = 0; r < S.R.size(); ++r) {
                ord[r] = (int32_t)r;
                for (auto& kv : S.R[r].kv) sum[r] += kv.second;
            }
            std::stable_sort(ord.begin(), ord.end(), [&](int32_t a, int32_t b) {
                return sum[a] != sum[b] ? sum[a] < sum[b] : S.R[a].inv < S.R[b].inv;
            });
            const int32_t n = (int32_t)ord.size();
            std::vector<GapOut> g(n);
            std::map<int32_t, std::vector<int32_t>> forced_in;   // transfer -> gaps forcing it in, ascending
            std::unique_ptr<Index> X;
            if (algo == RG_SEARCH) X.reset(new Index(S, keys));
            for (int32_t i = 0; i < n; ++i) {
                g[i] = decide_gap(S, keys, X.get(), S.R[ord[i]], i > 0 ? &S.R[ord[i - 1]] : nullptr, algo, max_nodes,
                                  o.nodes);
                codes.push_back(g[i].code);
                if (g[i].code == G_EXPLAINED) o.n_explained++;
                else if (g[i].code == G_UNDECIDED) o.n_undecided++;
                else o.count_by_kind[g[i].code - 1]++;
                for (int32_t t : g[i].forced) forced_in[t].push_back(i);
            }
            // the witness: the first violating gap, the smallest kind there, the smallest DOUBLE id there
            int32_t wgap = INT_MAX, wkind = 0, wt = -1;
            for (int32_t i = 0; i < n && wgap == INT_MAX; ++i)
                if (g[i].code == JTB_RG_KEY || g[i].code == JTB_RG_JOINT) { wgap = i; wkind = g[i].code; }
            for (auto& [t, gs] : forced_in) {
                if (gs.size() < 2) continue;
                o.count_by_kind[2]++;
                if (gs[1] < wgap || (gs[1] == wgap && wkind == JTB_RG_DOUBLE && S.T[t].id < S.T[wt].id)) {
                    wgap = gs[1];
                    wkind = JTB_RG_DOUBLE;
                    wt = t;
                }
            }
            if (wgap == INT_MAX) {
                o.valid = o.n_undecided ? JTB_UNKNOWN : JTB_VALID;
                continue;
            }
            o.valid = JTB_INVALID;
            o.kind = wkind;
            o.witness_index = S.R[ord[wgap]].comp_index;
            o.lower_index = wgap > 0 ? S.R[ord[wgap - 1]].comp_index : -1;
            o.n_eligible = g[wgap].n_eligible;
            if (wkind == JTB_RG_DOUBLE) {
                o.transfer_id = S.T[wt].id;
                o.other_index = S.R[ord[forced_in[wt][0]]].comp_index;
            } else {
                o.key = g[wgap].key;
                o.delta = g[wgap].delta;
            }
        }
    } catch (int) {
        return -2;
    }
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const jtb_rg_shard& o = shards[s] = tmp[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_explained += o.n_explained;
        out->n_unexplained += o.count_by_kind[0] + o.count_by_kind[1];
        out->n_double += o.count_by_kind[2];
        out->n_undecided += o.n_undecided;
        out->nodes += o.nodes;
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    if (per_gap) std::copy(codes.begin(), codes.end(), per_gap);
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
