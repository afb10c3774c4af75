// gaps_common.h — what the CPU oracles of the read-gap, the transfer-placement and the serial-witness checks share
// (TEST INFRASTRUCTURE ONLY): the shard parse, M(t) and A(t), a gap's subset-sum problem, its brute force, the
// library's search and the sweep structures of the gather; the transfer-placement check's windows, its gather and
// TP_SEARCH on one shard.  Its anonymous namespace gives each oracle a copy of its own.
#pragma once
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
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
    int32_t fate = -1, okcomp = NONE, cidx = -1;   // cidx: the :index of the completion
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
                    S.T[t].cidx = h->index[e];
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
[[maybe_unused]] bool brute(const Problem& pb, int32_t only, bool first, uint64_t& all) {
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

    // sol: the states of the first solution found
    bool dfs(const std::vector<int32_t>& F, std::vector<uint8_t>& st, const std::vector<int64_t>& base,
             std::vector<uint8_t>* sol) {
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
            if (!any) {
                if (sol) *sol = s2;
                return true;
            }
            if (dfs(F, s2, base, sol)) return true;
        }
        return false;
    }

    // root_key: the smallest key the root pruning found unreachable, -1; kept: candidates the root did not drop;
    // forced: the candidates a feasible root pruning forces in
    // root_st: the candidates' states after the root pruning, feasible or not
    // sol: EXPLAINED, the states of the first solution (IN: in it)
    Verdict run(int32_t& root_key, int32_t& kept, std::vector<int32_t>* forced = nullptr,
                std::vector<uint8_t>* root_st = nullptr, std::vector<uint8_t>* sol = nullptr) {
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
        if (root_st) *root_st = st;
        if (!ok) { root_key = pb.key[bad]; return UNEXPLAINED; }
        if (forced)
            for (int32_t c = 0; c < n; ++c)
                if (st[c] == IN) forced->push_back(c);
        std::vector<int32_t> F;
        for (int32_t c = 0; c < n; ++c)
            if (st[c] == UND) F.push_back(c);
        if (F.empty()) {
            if (sol) *sol = st;
            return EXPLAINED;
        }
        if (F.size() > (size_t)JTB_RG_MAX_FREE) return UNDECIDED;
        std::sort(F.begin(), F.end(), [&](int32_t x, int32_t y) {
            return pb.P[x].a != pb.P[y].a ? pb.P[x].a > pb.P[y].a : pb.P[x].id < pb.P[y].id;
        });
        std::vector<int64_t> base(pb.d.size());
        for (size_t k = 0; k < base.size(); ++k) base[k] = pb.d[k] - ins[k];   // ins: the forced-in of the root
        try {
            return dfs(F, st, base, sol) ? EXPLAINED : UNEXPLAINED;
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


// ---- the transfer-placement check (K12) ----------------------------------------------------------------------------
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

// The gather of gap i (upper read u, lower read l) into pb.P, with pb.d = Delta': round 0 every eligible transfer, a
// later round (or a witness round) only the in-window ones no gap owns; keep (may be null) drops more.  With cls (the
// class of each crashed transfer, -1 none) the crashed candidates of a class stop at cap = min over its observed keys
// of floor(Delta'_k / amount), the first ones in gather order.  false: past JTB_TP_MAX_GATHER.
bool gather_gap(const Shard& S, const Index& X, const std::vector<Window>& W, const std::vector<int32_t>& owner,
                const XRead& u, const XRead* l, int32_t i, int32_t round, Problem& pb,
                const std::function<bool(int32_t)>* keep = nullptr, const std::vector<int32_t>* cls = nullptr) {
    const int32_t K = (int32_t)pb.d.size();
    const int32_t ivl = l ? l->inv : -1;
    std::unordered_map<int32_t, int64_t> had;   // cls: gathered members per class
    auto take = [&](int32_t t) {
        const XTransfer& x = S.T[t];
        if (x.fate == JTB_T_FAIL || !(x.inv < u.comp) || !(x.A < u.comp) || x.M < ivl || x.amount <= 0) return true;
        if (round > 0 && !(W[t].win && W[t].lo <= i && i <= W[t].hi && owner[t] < 0)) return true;
        if (keep && !(*keep)(t)) return true;
        const int32_t jd = W[t].jd, jc = W[t].jc;
        if (jd < 0 && jc < 0) return true;
        if ((jd >= 0 && x.amount > pb.d[jd]) || (jc >= 0 && x.amount > pb.d[jc])) return true;
        if (cls && (*cls)[t] >= 0) {
            int64_t cap = INT64_MAX;
            if (jd >= 0) cap = pb.d[jd] / x.amount;
            if (jc >= 0) cap = std::min(cap, pb.d[jc] / x.amount);
            if (had[(*cls)[t]]++ >= cap) return true;
        }
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
    return fits;
}

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
    if (!gather_gap(S, X, W, owner, u, l, i, round, pb)) { code = G_UNDECIDED; g.inc = true; return latch(); }
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

// a shard's keys (sorted), whether some read misses one, and the order of its reads (K7's: sum of values, invocation)
[[maybe_unused]] void shard_order(const Shard& S, std::vector<int32_t>& keys, bool& partial, std::vector<int32_t>& ord) {
    keys.clear();
    for (auto& r : S.R)
        for (auto& kv : r.kv) keys.push_back(kv.first);
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    partial = false;
    for (auto& r : S.R) partial |= r.kv.size() < keys.size();
    ord.resize(S.R.size());
    std::vector<__int128> sum(S.R.size(), 0);
    for (size_t r = 0; r < S.R.size(); ++r) {
        ord[r] = (int32_t)r;
        for (auto& kv : S.R[r].kv) sum[r] += kv.second;
    }
    std::stable_sort(ord.begin(), ord.end(), [&](int32_t a, int32_t b) {
        return sum[a] != sum[b] ? sum[a] < sum[b] : S.R[a].inv < S.R[b].inv;
    });
}

// TP_SEARCH's state at the end of its rounds
struct TpState {
    std::vector<Window> W;
    std::vector<Gap> G;
    std::vector<int32_t> owner;
};

// TP_SEARCH on shard s (full-key, with reads, in the order ord): the rounds, the counts, the verdict and the witness
// into o; the windows, the gaps and the owners into T
[[maybe_unused]] void tp_search(const jtb_history* h, int32_t s, const Shard& S, const std::vector<int32_t>& keys,
                                const std::vector<int32_t>& ord, int64_t max_nodes, int32_t max_rounds,
                                jtb_tp_shard& o, TpState& T) {
    const int32_t n = (int32_t)ord.size(), K = (int32_t)keys.size(), nT = (int32_t)S.T.size();
    T.W = windows(S, keys, ord);
    const std::vector<Window>& W = T.W;
    auto upper = [&](int32_t i) -> const XRead& { return S.R[ord[i]]; };
    auto lower = [&](int32_t i) { return i > 0 ? &S.R[ord[i - 1]] : nullptr; };
    const Index X(S, keys);
    std::vector<Gap>& G = T.G;
    G.assign(n, Gap());
    for (auto& g : G) g.own.assign(K, 0);
    std::vector<int32_t>& owner = T.owner;
    owner.assign(nT, -1);
    std::vector<int32_t> dround(nT, -1), dg1(nT), dg2(nT), lround(nT, -1);
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
        return;
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

}  // namespace
