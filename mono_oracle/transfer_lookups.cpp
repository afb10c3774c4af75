// transfer_lookups.cpp — CPU oracle of the transfer-lookup check (TEST INFRASTRUCTURE ONLY; the library never calls it).
//
// Both deciders parse a shard the same plain way (reads and lookups paired with the latest invoke of their process,
// transfers with the next event of their process) and fill jtb_tl_shard exactly as jtb_check_transfer_lookups does.
// TL_LITERAL restates the definition: M(t) from every (lookup, record) pair, LOST / VANISHED from every (lookup,
// transfer) pair, the read rules from every (read, key, lookup) triple.
// TL_SWEEP makes one walk with hash maps: the earliest lookup returning each transfer, sorted M lists and counting for
// LOST / VANISHED, and per observed key a prefix max of S over lookups by completion and a suffix min by invocation.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../include/jtb_check.h"

namespace {

constexpr int TL_LITERAL = 0, TL_SWEEP = 1;
constexpr int32_t NONE = INT_MAX;

thread_local std::string g_err;

struct TRead {
    int32_t inv, comp, comp_index;
    std::vector<std::pair<int32_t, int64_t>> kv;   // sorted by key
};

struct TTransfer {
    int64_t id;
    int32_t debit, credit, amount;
    int32_t inv, inv_index;
    int32_t fate = -1, comp = -1, comp_index = -1;   // fate JTB_T_*, -1 = never completed
};

struct TLookup {
    int32_t inv, comp, comp_index;
    const int32_t* rec;   // n records of 5 int32
    int32_t n;
};

inline int64_t rec_id(const int32_t* r) { return (int64_t)(((uint64_t)(uint32_t)r[1] << 32) | (uint32_t)r[0]); }

struct Shard {
    std::vector<TRead> R;
    std::vector<TTransfer> T;
    std::vector<TLookup> L;   // in completion order
    std::unordered_map<int64_t, int32_t> tid;   // id -> transfer
};

int fail(const char* fmt, int32_t index, int64_t x = 0) {
    char buf[256];
    snprintf(buf, sizeof buf, fmt, index, (long long)x);
    g_err = buf;
    return -2;
}

int parse_shard(const jtb_history* h, int32_t s, Shard& S, int64_t& n_records) {
    const int64_t lo = h->shard_off[s], hi = h->shard_off[s + 1];
    std::unordered_map<int32_t, int32_t> last_inv;              // process -> position of its latest invoke
    std::unordered_map<int32_t, std::vector<size_t>> open;      // process -> its transfers awaiting a fate
    for (int64_t e = lo; e < hi; ++e) {
        const int32_t p = h->process[e], pos = (int32_t)(e - lo);
        if (p < 0) continue;
        auto ot = open.find(p);
        if (ot != open.end()) {
            if (h->type[e] != JTB_T_INVOKE)
                for (size_t t : ot->second) {
                    S.T[t].fate = h->type[e];
                    S.T[t].comp = pos;
                    S.T[t].comp_index = h->index[e];
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
                if (!S.tid.emplace(id, (int32_t)S.T.size()).second)
                    return fail("transfer at :index %d: id %lld is carried by two transfer invokes", h->index[e], id);
                TTransfer t;
                t.id = id; t.debit = r[2]; t.credit = r[3]; t.amount = r[4]; t.inv = pos; t.inv_index = h->index[e];
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
            S.L.push_back({inv, pos, h->index[e], h->payload + off, len / 5});
            continue;
        }
        if (h->f[e] != JTB_F_READ) continue;
        if (len % 3 != 0 || off < 0 || off + len > h->n_payload)
            return fail("read at :index %d: malformed payload", h->index[e]);
        TRead r;
        r.inv = inv;
        r.comp = pos;
        r.comp_index = h->index[e];
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

// What one op (an :ok lookup or read) violates: per kind whether it does and its smallest id (lookup kinds) or key
// (read kinds).
struct OpViol {
    bool any[JTB_TL_KINDS + 1] = {};
    int64_t min_id[JTB_TL_KINDS + 1];
    int32_t min_key[JTB_TL_KINDS + 1];
    OpViol() {
        for (int k = 0; k <= JTB_TL_KINDS; ++k) { min_id[k] = INT64_MAX; min_key[k] = INT_MAX; }
    }
    void id(int k, int64_t x) { any[k] = true; min_id[k] = std::min(min_id[k], x); }
    void key(int k, int32_t x) { any[k] = true; min_key[k] = std::min(min_key[k], x); }
    int code() const {
        for (int k = 1; k <= JTB_TL_KINDS; ++k)
            if (any[k]) return k;
        return 0;
    }
};

// records of lookup l: per-record kinds 1-4 and DUPLICATE (a record whose id an earlier record of l carries)
void record_kinds(const Shard& S, const TLookup& l, OpViol& v, jtb_tl_shard& o) {
    std::unordered_set<int64_t> seen;
    for (int32_t j = 0; j < l.n; ++j) {
        const int32_t* r = l.rec + 5 * j;
        const int64_t id = rec_id(r);
        if (!seen.insert(id).second) { o.count_by_kind[JTB_TL_DUPLICATE - 1]++; v.id(JTB_TL_DUPLICATE, id); }
        auto it = S.tid.find(id);
        if (it == S.tid.end()) { o.count_by_kind[JTB_TL_PHANTOM - 1]++; v.id(JTB_TL_PHANTOM, id); continue; }
        const TTransfer& t = S.T[it->second];
        if (t.debit != r[2] || t.credit != r[3] || t.amount != r[4]) {
            o.count_by_kind[JTB_TL_MISMATCH - 1]++;
            v.id(JTB_TL_MISMATCH, id);
        }
        if (t.fate == JTB_T_FAIL) { o.count_by_kind[JTB_TL_FAILED_VISIBLE - 1]++; v.id(JTB_TL_FAILED_VISIBLE, id); }
        if (t.inv > l.comp) { o.count_by_kind[JTB_TL_FUTURE - 1]++; v.id(JTB_TL_FUTURE, id); }
    }
}

// S_k(l) over the distinct ids of l (first record of each) for the keys in col
void lookup_sums(const TLookup& l, const std::unordered_map<int32_t, int32_t>& col, std::vector<int64_t>& S) {
    S.assign(col.size(), 0);
    std::unordered_set<int64_t> seen;
    for (int32_t j = 0; j < l.n; ++j) {
        const int32_t* r = l.rec + 5 * j;
        if (!seen.insert(rec_id(r)).second) continue;
        const int64_t ks[2] = {2 * (int64_t)r[2], 2 * (int64_t)r[3] + 1};
        for (int64_t k : ks) {
            if (k < INT_MIN || k > INT_MAX) continue;
            auto it = col.find((int32_t)k);
            if (it != col.end()) S[it->second] += r[4];
        }
    }
}

// M(t) and the lookup it came from (-1: the :ok completion, NONE: M is infinite)
struct MVal {
    int32_t m = NONE, from = NONE;
};

int lost_kind(const MVal& m) { return m.from == -1 ? JTB_TL_LOST : JTB_TL_VANISHED; }

// the witness of the op at completion position `at`; lookups: the smallest id of the kind and its related :index;
// reads: the smallest key, its value, the bound and the related lookup
struct Decided {
    std::vector<OpViol> lv, rv;   // per lookup, per read
    std::vector<MVal> M;          // per transfer
};

void fill_witness(const Shard& S, const Decided& D, const std::vector<std::vector<int64_t>>& Ssum,
                  const std::unordered_map<int32_t, int32_t>& col, jtb_tl_shard& o) {
    int32_t best = NONE, bl = -1, br = -1;
    for (size_t i = 0; i < S.L.size(); ++i)
        if (D.lv[i].code() && S.L[i].comp < best) { best = S.L[i].comp; bl = (int32_t)i; br = -1; }
    for (size_t i = 0; i < S.R.size(); ++i)
        if (D.rv[i].code() && S.R[i].comp < best) { best = S.R[i].comp; br = (int32_t)i; bl = -1; }
    if (best == NONE) return;
    o.valid = JTB_INVALID;
    if (bl >= 0) {
        const TLookup& l = S.L[bl];
        const int k = D.lv[bl].code();
        const int64_t id = D.lv[bl].min_id[k];
        o.witness_index = l.comp_index;
        o.kind = k;
        o.transfer_id = id;
        o.key = -1;
        o.related_index = -1;
        if (k == JTB_TL_PHANTOM || k == JTB_TL_DUPLICATE) return;
        const int32_t t = S.tid.at(id);
        if (k == JTB_TL_LOST) o.related_index = S.T[t].comp_index;
        else if (k == JTB_TL_VANISHED) o.related_index = S.L[D.M[t].from].comp_index;
        else o.related_index = S.T[t].inv_index;
        return;
    }
    const TRead& r = S.R[br];
    const int k = D.rv[br].code();
    const int32_t key = D.rv[br].min_key[k];
    int64_t v = 0;
    for (auto& kv : r.kv)
        if (kv.first == key) v = kv.second;
    const int32_t c = col.at(key);
    o.witness_index = r.comp_index;
    o.kind = k;
    o.key = key;
    o.value = v;
    o.transfer_id = 0;
    if (k == JTB_TL_READ_BELOW_LOOKUP) {
        int64_t bound = INT64_MIN;
        o.related_index = -1;
        for (size_t i = 0; i < S.L.size(); ++i)   // completion order
            if (S.L[i].comp < r.inv) {
                bound = std::max(bound, Ssum[i][c]);
                if (Ssum[i][c] > v && o.related_index < 0) o.related_index = S.L[i].comp_index;
            }
        o.bound = bound;
    } else {
        int64_t bound = INT64_MAX;
        int32_t first_inv = NONE;
        for (size_t i = 0; i < S.L.size(); ++i)
            if (S.L[i].inv > r.comp) {
                bound = std::min(bound, Ssum[i][c]);
                if (Ssum[i][c] < v && S.L[i].inv < first_inv) { first_inv = S.L[i].inv; o.related_index = S.L[i].comp_index; }
            }
        o.bound = bound;
    }
}

std::unordered_map<int32_t, int32_t> observed_keys(const Shard& S) {
    std::vector<int32_t> keys;
    for (auto& r : S.R)
        for (auto& kv : r.kv) keys.push_back(kv.first);
    std::sort(keys.begin(), keys.end());
    keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
    std::unordered_map<int32_t, int32_t> col;
    for (size_t i = 0; i < keys.size(); ++i) col.emplace(keys[i], (int32_t)i);
    return col;
}

void decide_literal(const Shard& S, jtb_tl_shard& o) {
    Decided D;
    D.lv.resize(S.L.size());
    D.rv.resize(S.R.size());
    for (size_t i = 0; i < S.L.size(); ++i) record_kinds(S, S.L[i], D.lv[i], o);
    // M(t) from every (lookup, record) pair
    D.M.resize(S.T.size());
    for (size_t t = 0; t < S.T.size(); ++t) {
        MVal& m = D.M[t];
        if (S.T[t].fate == JTB_T_OK) { m.m = S.T[t].comp; m.from = -1; }
        for (size_t i = 0; i < S.L.size(); ++i)
            for (int32_t j = 0; j < S.L[i].n; ++j)
                if (rec_id(S.L[i].rec + 5 * j) == S.T[t].id && S.L[i].comp < m.m) { m.m = S.L[i].comp; m.from = (int32_t)i; }
    }
    // every (lookup, transfer) pair
    for (size_t i = 0; i < S.L.size(); ++i)
        for (size_t t = 0; t < S.T.size(); ++t) {
            if (!(D.M[t].m < S.L[i].inv)) continue;
            bool in = false;
            for (int32_t j = 0; j < S.L[i].n && !in; ++j) in = rec_id(S.L[i].rec + 5 * j) == S.T[t].id;
            if (in) continue;
            const int k = lost_kind(D.M[t]);
            o.count_by_kind[k - 1]++;
            D.lv[i].id(k, S.T[t].id);
        }
    // every (read, key, lookup) triple
    const auto col = observed_keys(S);
    std::vector<std::vector<int64_t>> Ssum(S.L.size());
    for (size_t i = 0; i < S.L.size(); ++i) lookup_sums(S.L[i], col, Ssum[i]);
    for (size_t q = 0; q < S.R.size(); ++q)
        for (auto& [k, v] : S.R[q].kv) {
            bool below = false, above = false;
            for (size_t i = 0; i < S.L.size(); ++i) {
                const int64_t s = Ssum[i][col.at(k)];
                below |= S.L[i].comp < S.R[q].inv && v < s;
                above |= S.L[i].inv > S.R[q].comp && v > s;
            }
            if (below) { o.count_by_kind[JTB_TL_READ_BELOW_LOOKUP - 1]++; D.rv[q].key(JTB_TL_READ_BELOW_LOOKUP, k); }
            if (above) { o.count_by_kind[JTB_TL_READ_ABOVE_LOOKUP - 1]++; D.rv[q].key(JTB_TL_READ_ABOVE_LOOKUP, k); }
        }
    fill_witness(S, D, Ssum, col, o);
}

void decide_sweep(const Shard& S, jtb_tl_shard& o) {
    Decided D;
    const size_t nL = S.L.size(), nT = S.T.size();
    D.lv.resize(nL);
    D.rv.resize(S.R.size());
    for (size_t i = 0; i < nL; ++i) record_kinds(S, S.L[i], D.lv[i], o);
    // the earliest-completing lookup returning each transfer (lookups are in completion order)
    D.M.resize(nT);
    for (size_t t = 0; t < nT; ++t)
        if (S.T[t].fate == JTB_T_OK) { D.M[t].m = S.T[t].comp; D.M[t].from = -1; }
    std::vector<int32_t> first_lk(nT, -1);
    for (size_t i = 0; i < nL; ++i)
        for (int32_t j = 0; j < S.L[i].n; ++j) {
            auto it = S.tid.find(rec_id(S.L[i].rec + 5 * j));
            if (it != S.tid.end() && first_lk[it->second] < 0) first_lk[it->second] = (int32_t)i;
        }
    for (size_t t = 0; t < nT; ++t)
        if (first_lk[t] >= 0 && S.L[first_lk[t]].comp < D.M[t].m) { D.M[t].m = S.L[first_lk[t]].comp; D.M[t].from = first_lk[t]; }
    // need: transfers with M < inv(l), by kind (sorted M lists); have: l's distinct known ids with M < inv(l)
    std::vector<int32_t> mk[2];
    for (size_t t = 0; t < nT; ++t)
        if (D.M[t].m != NONE) mk[lost_kind(D.M[t]) - JTB_TL_LOST].push_back(D.M[t].m);
    for (auto& v : mk) std::sort(v.begin(), v.end());
    std::vector<int32_t> stamp(nT, -1);
    for (size_t i = 0; i < nL; ++i) {
        const TLookup& l = S.L[i];
        if (l.inv < 0) continue;
        int64_t have[2] = {0, 0};
        for (int32_t j = 0; j < l.n; ++j) {
            auto it = S.tid.find(rec_id(l.rec + 5 * j));
            if (it == S.tid.end() || stamp[it->second] == (int32_t)i) continue;
            stamp[it->second] = (int32_t)i;
            const MVal& m = D.M[it->second];
            if (m.m < l.inv) have[lost_kind(m) - JTB_TL_LOST]++;
        }
        for (int k = 0; k < 2; ++k) {
            const int64_t need = std::lower_bound(mk[k].begin(), mk[k].end(), l.inv) - mk[k].begin();
            if (need == have[k]) continue;
            o.count_by_kind[JTB_TL_LOST + k - 1] += need - have[k];
            int64_t min_id = INT64_MAX;   // the smallest missing id: one walk over the transfers
            for (size_t t = 0; t < nT; ++t)
                if (D.M[t].m < l.inv && lost_kind(D.M[t]) == JTB_TL_LOST + k && stamp[t] != (int32_t)i)
                    min_id = std::min(min_id, S.T[t].id);
            D.lv[i].id(JTB_TL_LOST + k, min_id);
        }
    }
    // reads: prefix max of S over lookups by completion, suffix min over lookups by invocation
    const auto col = observed_keys(S);
    const size_t K = col.size();
    std::vector<std::vector<int64_t>> Ssum(nL);
    for (size_t i = 0; i < nL; ++i) lookup_sums(S.L[i], col, Ssum[i]);
    std::vector<int64_t> pmax(nL * K), smin(nL * K);
    for (size_t i = 0; i < nL; ++i)
        for (size_t c = 0; c < K; ++c) pmax[i * K + c] = i ? std::max(pmax[(i - 1) * K + c], Ssum[i][c]) : Ssum[i][c];
    std::vector<int32_t> by_inv;
    for (size_t i = 0; i < nL; ++i)
        if (S.L[i].inv >= 0) by_inv.push_back((int32_t)i);
    std::stable_sort(by_inv.begin(), by_inv.end(), [&](int32_t a, int32_t b) { return S.L[a].inv < S.L[b].inv; });
    std::vector<int32_t> inv_sorted(by_inv.size());
    for (size_t j = by_inv.size(); j-- > 0;) {
        inv_sorted[j] = S.L[by_inv[j]].inv;
        for (size_t c = 0; c < K; ++c)
            smin[j * K + c] = j + 1 < by_inv.size() ? std::min(smin[(j + 1) * K + c], Ssum[by_inv[j]][c])
                                                   : Ssum[by_inv[j]][c];
    }
    std::vector<int32_t> comps(nL);
    for (size_t i = 0; i < nL; ++i) comps[i] = S.L[i].comp;
    for (size_t q = 0; q < S.R.size(); ++q) {
        const TRead& r = S.R[q];
        const size_t nb = std::lower_bound(comps.begin(), comps.end(), r.inv) - comps.begin();   // comp < inv
        const size_t ja = std::upper_bound(inv_sorted.begin(), inv_sorted.end(), r.comp) - inv_sorted.begin();
        for (auto& [k, v] : r.kv) {
            const size_t c = col.at(k);
            if (r.inv >= 0 && nb > 0 && v < pmax[(nb - 1) * K + c]) {
                o.count_by_kind[JTB_TL_READ_BELOW_LOOKUP - 1]++;
                D.rv[q].key(JTB_TL_READ_BELOW_LOOKUP, k);
            }
            if (ja < by_inv.size() && v > smin[ja * K + c]) {
                o.count_by_kind[JTB_TL_READ_ABOVE_LOOKUP - 1]++;
                D.rv[q].key(JTB_TL_READ_ABOVE_LOOKUP, k);
            }
        }
    }
    fill_witness(S, D, Ssum, col, o);
}

}  // namespace

extern "C" {

const char* jtbm_tl_last_error(void) { return g_err.c_str(); }

int jtbm_check_transfer_lookups(const jtb_history* h, int32_t flags, int32_t algo, jtb_tl_shard* shards,
                                jtb_tl_result* out) {
    const auto t0 = std::chrono::steady_clock::now();
    if (flags != 0) { g_err = "flags must be 0 (reserved)"; return -2; }
    memset(out, 0, sizeof *out);
    int64_t n_records = 0, n_reads = 0;
    std::vector<jtb_tl_shard> tmp(h->n_shards);
    for (int32_t s = 0; s < h->n_shards; ++s) {
        Shard S;
        if (int rc = parse_shard(h, s, S, n_records)) return rc;
        n_reads += (int64_t)S.R.size();
        if (n_reads > INT_MAX) { g_err = "more than 2^31-1 reads"; return -2; }
        jtb_tl_shard& o = tmp[s];
        memset(&o, 0, sizeof o);
        o.n_lookups = (int32_t)S.L.size();
        for (auto& l : S.L) o.n_records += l.n;
        o.n_transfers = (int32_t)S.T.size();
        o.n_reads = (int32_t)S.R.size();
        o.witness_index = o.key = o.related_index = -1;
        if (algo == TL_SWEEP) decide_sweep(S, o);
        else decide_literal(S, o);
    }
    for (int32_t s = 0; s < h->n_shards; ++s) {
        const jtb_tl_shard& o = shards[s] = tmp[s];
        out->n_lookups += o.n_lookups;
        out->n_records += o.n_records;
        out->n_transfers += o.n_transfers;
        out->n_reads += o.n_reads;
        for (int k = 0; k < JTB_TL_KINDS; ++k) out->n_violations += o.count_by_kind[k];
        out->valid = std::max(out->valid, o.valid);
        if (o.valid != JTB_VALID) out->n_failures++;
    }
    out->seconds_total = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    return 0;
}

}  // extern "C"
