// read_explanations.cpp — CPU oracle of the read-explanation check (TEST INFRASTRUCTURE ONLY; the library never calls
// it).
//
// Both deciders parse a shard the way the transfer-lookup oracle does (reads and lookups paired with the latest invoke
// of their process, every [:t ...] micro-op a transfer paired with the next event of its process), classify every
// transfer for every :ok read as must / cannot / may, and fill jtb_rx_shard as jtb_check_read_explanations does.
// RX_BRUTE is the definition: every subset of the "may" transfers, no budget (tiny histories only).
// RX_SEARCH is the library's decision: the same caps, the root pruning fixpoint in Jacobi rounds, at most 64 free
// candidates in the canonical order (amount descending, then id), a depth-first search including before excluding,
// the same fixpoint at every node, and the node budget.  Node counts are the library's.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../include/jtb_check.h"

namespace {

constexpr int RX_BRUTE = 0, RX_SEARCH = 1;
constexpr int32_t NONE = INT_MAX;
// per-read codes of the optional per-read output
constexpr int8_t R_EXPLAINED = 0, R_UNDECIDED = 3;

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
    int32_t a, jd, jc;   // jd / jc: index of the debit / credit key among the read's sorted keys, -1 unobserved
};

// One read's subset-sum problem: candidates, d per key (the read's sorted keys).
struct Problem {
    std::vector<Cand> P;
    std::vector<int64_t> d;
    std::vector<int32_t> key;
    std::vector<int64_t> must_sum;
};

int32_t key_index(const XRead& r, int64_t key) {
    auto it = std::lower_bound(r.kv.begin(), r.kv.end(), std::make_pair((int32_t)std::min<int64_t>(key, INT_MAX),
                                                                        INT64_MIN));
    return it != r.kv.end() && it->first == key ? (int32_t)(it - r.kv.begin()) : -1;
}

// the "may" test of a transfer that is not must for r
inline bool may(const XTransfer& t, const XRead& r) {
    return t.fate != JTB_T_FAIL && t.inv < r.comp && t.A < r.comp && t.amount > 0;
}

// RX_BRUTE: every transfer against the definition
void build_literal(const Shard& S, const XRead& r, Problem& pb) {
    for (auto& t : S.T) {
        const int32_t jd = key_index(r, 2 * (int64_t)t.debit), jc = key_index(r, 2 * (int64_t)t.credit + 1);
        if (t.M < r.inv) {
            if (jd >= 0) pb.must_sum[jd] += t.amount;
            if (jc >= 0) pb.must_sum[jc] += t.amount;
        } else if (may(t, r) && (jd >= 0 || jc >= 0)) {
            pb.P.push_back({t.id, t.amount, jd, jc});
        }
    }
}

// RX_SEARCH's sweep structures: per key the (M, running sum) list, the :ok transfers in invocation order (the order of
// S.T) with the running max of their completions, the crashed (:info, never completed) ones in invocation order
struct Index {
    std::unordered_map<int64_t, std::vector<std::pair<int32_t, int64_t>>> msum;
    std::vector<int32_t> ok, ok_inv, ok_pmax, crashed, crashed_inv;
    explicit Index(const Shard& S) {
        for (size_t i = 0; i < S.T.size(); ++i) {
            const XTransfer& t = S.T[i];
            msum[2 * (int64_t)t.debit].push_back({t.M, t.amount});
            msum[2 * (int64_t)t.credit + 1].push_back({t.M, t.amount});
            if (t.fate == JTB_T_OK) {
                ok.push_back((int32_t)i);
                ok_inv.push_back(t.inv);
                ok_pmax.push_back(std::max(ok_pmax.empty() ? INT_MIN : ok_pmax.back(), t.okcomp));
            } else if (t.fate != JTB_T_FAIL) {
                crashed.push_back((int32_t)i);
                crashed_inv.push_back(t.inv);
            }
        }
        for (auto& [k, v] : msum) {
            std::sort(v.begin(), v.end());
            for (size_t j = 1; j < v.size(); ++j) v[j].second += v[j - 1].second;
        }
    }
};

// false: more "may" transfers than the gather cap
bool build_sweep(const Shard& S, const Index& X, const XRead& r, Problem& pb) {
    for (size_t j = 0; j < r.kv.size(); ++j) {
        auto it = X.msum.find(r.kv[j].first);
        if (it == X.msum.end()) continue;
        auto e = std::lower_bound(it->second.begin(), it->second.end(), std::make_pair(r.inv, INT64_MIN));
        if (e != it->second.begin()) pb.must_sum[j] = (e - 1)->second;
    }
    auto take = [&](int32_t i) {
        const XTransfer& t = S.T[i];
        if (t.M < r.inv || !may(t, r)) return true;
        const int32_t jd = key_index(r, 2 * (int64_t)t.debit), jc = key_index(r, 2 * (int64_t)t.credit + 1);
        if (jd < 0 && jc < 0) return true;
        pb.P.push_back({t.id, t.amount, jd, jc});
        return pb.P.size() <= (size_t)JTB_RX_MAX_GATHER;
    };
    // :ok transfers invoked before r completed, back to the last one whose running max completion is before r's
    // invocation (every earlier one completed before it, so is must)
    for (int64_t j = std::lower_bound(X.ok_inv.begin(), X.ok_inv.end(), r.comp) - X.ok_inv.begin() - 1;
         j >= 0 && X.ok_pmax[j] >= r.inv; --j)
        if (!take(X.ok[j])) return false;
    const int64_t bc = std::lower_bound(X.crashed_inv.begin(), X.crashed_inv.end(), r.comp) - X.crashed_inv.begin();
    for (int64_t j = 0; j < bc; ++j)
        if (!take(X.crashed[j])) return false;
    return true;
}

int32_t count_must(const Shard& S, const XRead& r) {
    int32_t n = 0;
    for (auto& t : S.T)
        n += t.M < r.inv && (key_index(r, 2 * (int64_t)t.debit) >= 0 || key_index(r, 2 * (int64_t)t.credit + 1) >= 0);
    return n;
}

// ---- RX_BRUTE ----------------------------------------------------------------------------------------------------
// is there X within P with sum d on every key (only >= 0: on that key alone)?
bool brute(const Problem& pb, int32_t only) {
    const size_t n = pb.P.size(), K = pb.d.size();
    if (n > 24) { g_err = "RX_BRUTE: more than 24 candidates"; throw 1; }
    std::vector<int64_t> s(K);
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
        if (ok) return true;
    }
    return false;
}

// ---- RX_SEARCH ---------------------------------------------------------------------------------------------------
enum { UND = 0, IN = 1, OUT = 2 };
enum Verdict { EXPLAINED, UNEXPLAINED, UNDECIDED };

struct Search {
    const Problem& pb;
    int32_t only;
    int64_t max_nodes, nodes = 0;
    std::vector<int64_t> ins, av;

    Search(const Problem& p, int32_t o, int64_t mx) : pb(p), only(o), max_nodes(mx), ins(p.d.size()), av(p.d.size()) {}

    int32_t rel(int32_t j) const { return only < 0 || j == only ? j : -1; }

    // one fixpoint of Jacobi rounds over candidates `ids` (state st, base need `base`); false when infeasible, with
    // bad = the smallest infeasible key index of that round
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

    // root_key: the smallest key the root pruning found unreachable, -1; kept: candidates the root did not drop
    Verdict run(int32_t& root_key, int32_t& kept) {
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
        std::vector<int32_t> F;
        for (int32_t c = 0; c < n; ++c)
            if (st[c] == UND) F.push_back(c);
        if (F.empty()) return EXPLAINED;
        if (F.size() > (size_t)JTB_RX_MAX_FREE) return UNDECIDED;
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

struct ReadOut {
    int8_t code = R_EXPLAINED;
    int32_t key = -1, n_may = 0;
    int64_t value = 0, must_sum = 0;
};

ReadOut decide_read(const Shard& S, const Index* X, const XRead& r, int64_t max_nodes, int64_t& nodes) {
    ReadOut o;
    if (X && r.kv.size() > (size_t)JTB_RX_MAX_KEYS) { o.code = R_UNDECIDED; return o; }
    Problem pb;
    const int32_t K = (int32_t)r.kv.size();
    pb.key.resize(K);
    pb.must_sum.assign(K, 0);
    pb.d.resize(K);
    for (int32_t j = 0; j < K; ++j) pb.key[j] = r.kv[j].first;
    if (!X) build_literal(S, r, pb);
    else if (!build_sweep(S, *X, r, pb)) { o.code = R_UNDECIDED; return o; }
    for (int32_t j = 0; j < K; ++j) pb.d[j] = r.kv[j].second - pb.must_sum[j];
    if (!X) {
        o.n_may = (int32_t)pb.P.size();
        if (brute(pb, -1)) return o;
        o.code = JTB_RX_JOINT;
        for (int32_t k = 0; k < K; ++k)
            if (!brute(pb, k)) { o.code = JTB_RX_KEY; o.key = pb.key[k]; break; }
    } else {
        Search s(pb, -1, max_nodes);
        int32_t root_key, kept;
        const Verdict v = s.run(root_key, kept);
        nodes += s.nodes;
        o.n_may = kept;
        if (v == EXPLAINED) return o;
        if (v == UNDECIDED) { o.code = R_UNDECIDED; return o; }
        o.code = JTB_RX_JOINT;
        o.key = root_key;
        for (int32_t k = 0; k < K; ++k) {
            Search sk(pb, k, max_nodes);
            int32_t rk, kp;
            const Verdict vk = sk.run(rk, kp);
            nodes += sk.nodes;
            if (vk == UNEXPLAINED) { o.code = JTB_RX_KEY; o.key = pb.key[k]; break; }
        }
    }
    if (o.code == JTB_RX_KEY) {
        const int32_t k = key_index(r, o.key);
        o.value = r.kv[k].second;
        o.must_sum = pb.must_sum[k];
    }
    return o;
}

}  // namespace

extern "C" {

const char* jtbm_rx_last_error(void) { return g_err.c_str(); }

// per_read (may be NULL): one code per :ok read in shard-major completion order: 0 explained, 1 KEY, 2 JOINT,
// 3 undecided
int jtbm_check_read_explanations(const jtb_history* h, int64_t max_nodes, int32_t flags, int32_t algo,
                                 jtb_rx_shard* shards, jtb_rx_result* out, int8_t* per_read) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    if (max_nodes <= 0) max_nodes = JTB_RX_DEFAULT_MAX_NODES;
    memset(out, 0, sizeof *out);
    int64_t n_records = 0, n_reads = 0;
    std::vector<jtb_rx_shard> tmp(h->n_shards);
    std::vector<int8_t> codes;
    try {
        for (int32_t s = 0; s < h->n_shards; ++s) {
            Shard S;
            if (int rc = parse_shard(h, s, S, n_records)) return rc;
            n_reads += (int64_t)S.R.size();
            if (n_reads > INT_MAX) { g_err = "more than 2^31-1 reads"; return -2; }
            classify_inputs(S);
            jtb_rx_shard& o = tmp[s];
            memset(&o, 0, sizeof o);
            o.valid = JTB_VALID;
            o.n_reads = (int32_t)S.R.size();
            o.n_transfers = (int32_t)S.T.size();
            o.witness_index = o.key = -1;
            std::unique_ptr<Index> X;
            if (algo == RX_SEARCH) X.reset(new Index(S));
            for (auto& r : S.R) {
                const ReadOut ro = decide_read(S, X.get(), r, max_nodes, o.nodes);
                codes.push_back(ro.code);
                if (ro.code == R_EXPLAINED) { o.n_explained++; continue; }
                if (ro.code == R_UNDECIDED) { o.n_undecided++; continue; }
                o.count_by_kind[ro.code - 1]++;
                if (o.witness_index >= 0) continue;   // reads are in completion order: the first is the earliest
                o.witness_index = r.comp_index;
                o.kind = ro.code;
                o.key = ro.key;
                o.n_must = count_must(S, r);
                o.n_may = ro.n_may;
                o.value = ro.value;
                o.must_sum = ro.must_sum;
            }
            o.valid = o.witness_index >= 0 ? JTB_INVALID : o.n_undecided ? JTB_UNKNOWN : JTB_VALID;
        }
    } catch (int) {
        return -2;
    }
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const jtb_rx_shard& o = shards[s] = tmp[s];
        out->n_reads += o.n_reads;
        out->n_transfers += o.n_transfers;
        out->n_explained += o.n_explained;
        out->n_unexplained += o.count_by_kind[0] + o.count_by_kind[1];
        out->n_undecided += o.n_undecided;
        out->nodes += o.nodes;
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    if (per_read) std::copy(codes.begin(), codes.end(), per_read);
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
