// hostwalk_dups.cpp — TEST INFRASTRUCTURE / MEASUREMENT (not part of libjtb_check.so, never loaded by the product).
//
// The level-synchronous host walk of hostwalk.cpp (walk_bfs: the product's expansion core, jtb_expand.h, breadth-first
// with a visited set that lives for one level), with per-level statistics of where the duplicates of a level are:
// for every level, the parents expanded, the children generated (every child that does not complete its shard — the
// ones the device probes the window with), the new configurations, and for each window size W the children that
// repeat a key already generated from the same block of W consecutive parents (blocks aligned at multiples of W, in
// the walk's order: a tile filter over tiles of W parents drops exactly these).  The search itself is walk_bfs's:
// same configurations, same verdict.
#include <cstring>
#include <string>
#include <unordered_set>
#include <vector>

#include "../../jepsen_tigerbeetle_b200/csrc/jtb_expand.h"

using namespace jtb;

namespace {

constexpr int MAX_WIN = 4;

// stats: per level, 3 + n_win words: parents, children, new, dups within W_0 .. W_{n_win-1}
template <int MODEL, int KW, bool EAGER>
void walk_dups(const Prepared& P, const jtb_model* m, unsigned long long max_configs, int n_shards, int32_t* valid,
               unsigned long long* configs_out, const int* win, int n_win, unsigned long long* stats, int cap,
               int* n_levels_out) {
    ExpandTables T{P.rows.data(), P.classes.data(), P.cls_inv_pos.data(), P.row_words, P.sum_off};
    struct Entry { uint64_t w[KW]; int32_t bal[8]; };
    std::vector<Entry> cur, nxt;
    std::vector<char> found(n_shards, 0);
    for (int s = 0; s < n_shards; ++s) {
        if (P.shard_cause[s]) { valid[s] = JTB_UNKNOWN; found[s] = 2; continue; }
        if (P.rank_base[s + 1] == P.rank_base[s]) { valid[s] = JTB_VALID; found[s] = 2; continue; }
        Entry e0{};
        e0.w[0] = XKEY_VALID | ((uint64_t)(uint32_t)P.rank_base[s] << 32) |
                  ((MODEL == JTB_MODEL_BANK || MODEL == JTB_MODEL_SET) ? 0ull : (uint64_t)(uint32_t)m->init_value);
        for (int i = 0; i < 8; ++i) e0.bal[i] = m->init_balance[i];
        cur.push_back(e0);
    }
    unsigned long long configs = 0;
    bool budget_hit = false;
    int level = 0;
    const int row = 3 + n_win;
    while (!cur.empty() && !budget_hit) {
        std::unordered_set<std::string> seen;   // this level only
        std::unordered_set<std::string> block[MAX_WIN];
        unsigned long long children = 0, dups[MAX_WIN] = {0};
        nxt.clear();
        size_t parents = 0;
        for (const Entry& e : cur) {
            for (int x = 0; x < n_win; ++x)
                if (parents % (size_t)win[x] == 0) block[x].clear();
            ++parents;
            Expander<MODEL, KW, EAGER> X;
            for (int i = 0; i < KW; ++i) X.w[i] = e.w[i];
            for (int i = 0; i < 8; ++i) X.bal[i] = e.bal[i];
            const int s = X.load_header(T);
            X.begin(T, !found[s]);
            Child<KW> ch;
            while (X.next(T, m->negative_balances_ok != 0, ch)) {
                if (ch.done) { found[s] = 1; break; }
                std::string key(reinterpret_cast<const char*>(ch.w), sizeof ch.w);
                ++children;
                for (int x = 0; x < n_win; ++x)
                    if (!block[x].insert(key).second) ++dups[x];
                if (!seen.insert(key).second) continue;
                ++configs;
                Entry c;
                for (int i = 0; i < KW; ++i) c.w[i] = ch.w[i];
                for (int i = 0; i < 8; ++i) c.bal[i] = e.bal[i];
                if (ch.amt) { c.bal[ch.d] -= ch.amt; c.bal[ch.c] += ch.amt; }
                nxt.push_back(c);
            }
            if (max_configs && configs >= max_configs) { budget_hit = true; break; }
        }
        if (level < cap) {
            unsigned long long* r = stats + (size_t)level * row;
            r[0] = parents; r[1] = children; r[2] = nxt.size();
            for (int x = 0; x < n_win; ++x) r[3 + x] = dups[x];
        }
        ++level;
        cur.swap(nxt);
    }
    *n_levels_out = level;
    for (int s = 0; s < n_shards; ++s) {
        if (found[s] == 2) continue;
        valid[s] = found[s] ? JTB_VALID : budget_hit ? JTB_UNKNOWN : JTB_INVALID;
    }
    *configs_out = configs;
}

template <int MODEL>
int dups_kw(int kw, bool eager, const Prepared& P, const jtb_model* m, unsigned long long mc, int ns, int32_t* v,
            unsigned long long* c, const int* win, int n_win, unsigned long long* stats, int cap, int* nl) {
    switch (kw) {
    case 2: if (eager) walk_dups<MODEL, 2, true>(P, m, mc, ns, v, c, win, n_win, stats, cap, nl);
            else walk_dups<MODEL, 2, false>(P, m, mc, ns, v, c, win, n_win, stats, cap, nl);
            return 0;
    case 4: if (eager) walk_dups<MODEL, 4, true>(P, m, mc, ns, v, c, win, n_win, stats, cap, nl);
            else walk_dups<MODEL, 4, false>(P, m, mc, ns, v, c, win, n_win, stats, cap, nl);
            return 0;
    case 8: if (eager) walk_dups<MODEL, 8, true>(P, m, mc, ns, v, c, win, n_win, stats, cap, nl);
            else walk_dups<MODEL, 8, false>(P, m, mc, ns, v, c, win, n_win, stats, cap, nl);
            return 0;
    }
    return -1;
}

}  // namespace

extern "C" int jtb_hostwalk_dups(const jtb_history* h, const jtb_model* m, int eager, unsigned long long max_configs,
                                 int32_t* valid, unsigned long long* configs, const int* windows, int n_windows,
                                 unsigned long long* stats, int cap, int* n_levels) {
    if (n_windows < 0 || n_windows > MAX_WIN) return -4;
    for (int x = 0; x < n_windows; ++x)
        if (windows[x] < 1) return -4;
    Prepared P;
    if (!prepare(h, m, P)) return -3;
    for (int s = 0; s < h->n_shards; ++s) valid[s] = JTB_UNKNOWN;
    const int ns = h->n_shards;
    switch (m->kind) {
    case JTB_MODEL_BANK: return dups_kw<JTB_MODEL_BANK>(P.key_words, eager != 0, P, m, max_configs, ns, valid, configs, windows, n_windows, stats, cap, n_levels);
    case JTB_MODEL_SET: return dups_kw<JTB_MODEL_SET>(P.key_words, eager != 0, P, m, max_configs, ns, valid, configs, windows, n_windows, stats, cap, n_levels);
    case JTB_MODEL_REGISTER:
    case JTB_MODEL_CAS_REGISTER:
        return dups_kw<JTB_MODEL_CAS_REGISTER>(P.key_words, eager != 0, P, m, max_configs, ns, valid, configs, windows, n_windows, stats, cap, n_levels);
    }
    return -2;
}
