// Host emulation of the level engine's beam on the DEVICE's expansion core (csrc/jtb_expand.h + csrc/jtb_prep.cpp):
//   g++ -O2 -std=c++17 -fPIC -shared -I. -DCMAX=15 -o /tmp/libbeam.so scripts/experiments/beam_emulation.cpp \
//       jepsen_tigerbeetle_b200/csrc/jtb_prep.cpp ;  python scripts/experiments/beam_emulation.py
// policy 0 = (rank desc, crashed asc) exact top-W, 1 = (crashed asc, rank desc) exact top-W, 2 = the device's binned keys
// relative to the previous level's best + pseudo-random share of the boundary bin.  BEAM_LAZY=1 (bank): crashed
// transfers only when they move the balances towards a pending read.
// experiment: level-synchronous BEAM (keep the W best configurations of every level: furthest rank first, then fewest
// crashed ops consumed; no backlog) — does it find the linearization of crash-heavy VALID histories, at which W?
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_set>
#include <vector>
#include "jepsen_tigerbeetle_b200/csrc/jtb_expand.h"
using namespace jtb;
template <int MODEL, int KW, bool EAGER>
static int beam(const Prepared& P, const jtb_model* m, int W, int policy, unsigned long long* out) {
    ExpandTables T{P.rows.data(), P.classes.data(), P.cls_inv_pos.data(), P.row_words, P.sum_off};
    struct Entry { uint64_t w[KW]; int crashed; int32_t bal[8]; };
    std::vector<Entry> cur, nxt; Entry e0{}; e0.w[0] = XKEY_VALID | ((MODEL == JTB_MODEL_BANK) ? 0ull : (uint64_t)(uint32_t)m->init_value); for (int i = 0; i < 8; ++i) e0.bal[i] = m->init_balance[i]; cur.push_back(e0);
    unsigned long long configs = 0, levels = 0, maxw = 0;
    int in_min_c = 0, in_max_r = 0;
    while (!cur.empty() && configs < 40000000ull) {
        std::unordered_set<std::string> seen; nxt.clear();
        for (const Entry& e : cur) {
            Expander<MODEL, KW, EAGER> X;
            for (int k = 0; k < KW; ++k) X.w[k] = e.w[k];
            for (int k = 0; k < 8; ++k) X.bal[k] = e.bal[k];
            X.load_header(T); X.begin(T, true);
            Child<KW> ch;
            uint64_t todo = X.todo;
            auto take = [&](bool crashed) -> bool {
                if (ch.done) return true;
                std::string key((const char*)ch.w, sizeof ch.w);
                if (!seen.insert(key).second) return false;
                ++configs;
                Entry c; for (int k = 0; k < KW; ++k) c.w[k] = ch.w[k];
                c.crashed = e.crashed + (crashed ? 1 : 0);
                for (int k = 0; k < 8; ++k) c.bal[k] = e.bal[k];
                if (ch.amt) { c.bal[ch.d] -= ch.amt; c.bal[ch.c] += ch.amt; }
                nxt.push_back(c);
                return false;
            };
            while (todo) { int t = __builtin_ctzll(todo); todo &= todo - 1; if (X.child_slot(T, t, true, ch) && take(false)) goto found; }
            if (X.cls_i == 0) {
                // bank: "lazy crashed transfers" — only those that move the balances towards a pending read
                int32_t Er[64][8]; int nr = 0;
                if (MODEL == JTB_MODEL_BANK && getenv("BEAM_LAZY")) {
                    const int32_t* row = X.row;
                    uint64_t cand, rdm; memcpy(&cand, row + 14, 8); memcpy(&rdm, row + 16, 8);
                    uint64_t rds = cand & rdm & ~X.w[1];
                    while (rds) { int t = __builtin_ctzll(rds); rds &= rds - 1; const int32_t* cell = row + ROW_EXTRA + t * 12; for (int k = 0; k < 8; ++k) Er[nr][k] = cell[4 + k]; ++nr; }
                }
                for (int ci = 0; ci < X.ncls; ++ci) {
                    if (!X.child_class(T, ci, true, ch)) continue;
                    if (MODEL == JTB_MODEL_BANK && getenv("BEAM_LAZY")) {
                        bool useful = false;
                        for (int r = 0; r < nr && !useful; ++r) useful = Er[r][ch.d] < X.bal[ch.d] && Er[r][ch.c] > X.bal[ch.c];
                        if (!useful) continue;
                    }
                    if (take(true)) goto found;
                }
            }
        }
        ++levels; maxw = std::max<unsigned long long>(maxw, nxt.size());
        if (policy == 2) {
            // emulate the device: key relative to the INPUT level's trackers (min crashed, max rank over all appended)
            std::vector<int> keys(nxt.size());
            std::vector<unsigned> hist(64 * 64, 0);
            for (size_t i = 0; i < nxt.size(); ++i) {
                int c = nxt[i].crashed - in_min_c, r = in_max_r + 2 - (int)((nxt[i].w[0] >> 32) & XRANK_MASK);
                c = c < 0 ? 0 : (c > CMAX ? CMAX : c); r = r < 0 ? 0 : (r > 63 ? 63 : r);
                keys[i] = c * 64 + r; hist[keys[i]]++;
            }
            int out_min_c = 1 << 30, out_max_r = -1;
            for (auto& e : nxt) { out_min_c = std::min(out_min_c, e.crashed); out_max_r = std::max(out_max_r, (int)((e.w[0] >> 32) & XRANK_MASK)); }
            if ((int)nxt.size() > W) {
                unsigned long long run = 0; int thr = 64 * 64 - 1;
                for (int b = 0; b < 64 * 64; ++b) { run += hist[b]; if (run >= (unsigned long long)W) { thr = b; break; } }
                std::vector<Entry> kept;
                const unsigned long long below = run - hist[thr];
                const unsigned frac = (unsigned)(((unsigned long long)W - below) * 1024ull / hist[thr]) + 1;   // of 1024
                for (size_t i = 0; i < nxt.size(); ++i) {
                    if (keys[i] < thr) kept.push_back(nxt[i]);
                    else if (keys[i] == thr) {
                        uint64_t hsh = 0x9E3779B97F4A7C15ull;
                        for (int k = 0; k < KW; ++k) { hsh ^= nxt[i].w[k]; hsh *= 0xFF51AFD7ED558CCDull; hsh ^= hsh >> 32; }
                        if ((hsh & 1023) < frac) kept.push_back(nxt[i]);
                    }
                }
                nxt.swap(kept);
            }
            if (getenv("BEAM_TRACE") && (levels < 40 || levels % 25 == 0)) fprintf(stderr, "[emu] level %llu n_out %zu(kept) min_c %d max_r %d\n", levels, nxt.size(), out_min_c, out_max_r);
            in_min_c = out_min_c; in_max_r = out_max_r;
        } else if ((int)nxt.size() > W) {
            auto rank = [](const Entry& x) { return (uint32_t)((x.w[0] >> 32) & XRANK_MASK); };
            if (policy == 0) std::nth_element(nxt.begin(), nxt.begin() + W, nxt.end(), [&](const Entry& a, const Entry& b) {
                    if (rank(a) != rank(b)) return rank(a) > rank(b); return a.crashed < b.crashed; });
            else std::nth_element(nxt.begin(), nxt.begin() + W, nxt.end(), [&](const Entry& a, const Entry& b) {
                    if (a.crashed != b.crashed) return a.crashed < b.crashed; return rank(a) > rank(b); });
            nxt.resize(W);
        }
        cur.swap(nxt);
    }
    out[0] = 0; out[1] = configs; out[2] = levels; out[3] = maxw; return 0;
found:
    out[0] = 1; out[1] = configs; out[2] = levels; out[3] = maxw; return 0;
}
extern "C" int beam_run(const jtb_history* h, const jtb_model* m, int W, int policy, int eager, unsigned long long* out) {
    Prepared P; if (!prepare(h, m, P)) return -1;
    out[4] = P.key_words;
    if (m->kind == JTB_MODEL_BANK) {
        switch (P.key_words) {
        case 2: return beam<JTB_MODEL_BANK, 2, true>(P, m, W, policy, out);
        case 4: return beam<JTB_MODEL_BANK, 4, true>(P, m, W, policy, out);
        case 8: return beam<JTB_MODEL_BANK, 8, true>(P, m, W, policy, out);
        }
    }
    switch (P.key_words) {
    case 2: return eager ? beam<JTB_MODEL_CAS_REGISTER, 2, true>(P, m, W, policy, out) : beam<JTB_MODEL_CAS_REGISTER, 2, false>(P, m, W, policy, out);
    case 4: return eager ? beam<JTB_MODEL_CAS_REGISTER, 4, true>(P, m, W, policy, out) : beam<JTB_MODEL_CAS_REGISTER, 4, false>(P, m, W, policy, out);
    case 8: return eager ? beam<JTB_MODEL_CAS_REGISTER, 8, true>(P, m, W, policy, out) : beam<JTB_MODEL_CAS_REGISTER, 8, false>(P, m, W, policy, out);
    }
    return -2;
}
