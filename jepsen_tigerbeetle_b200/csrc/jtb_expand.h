// jtb_expand.h — ONE thread expands ONE configuration: the per-thread core of the level engine (jtb_level.cuh).
//
// Replaces the inner loop of knossos.wgl/analysis (SURVEY.md A.5: `step` over every call entry that may be
// linearized next, then `cache.add`).  The same code compiles for the device (inlined into the persistent kernel) and
// for the host (tests/native/hostwalk.cpp drives it with a std::unordered_set as the visited set, so the candidate
// rules, the frontier advance and the eager-read rule are checked against the oracle on the CPU tier too).
//
// A configuration is (key words w[KW], bank balances).  Children are produced one at a time by next():
//   1. begin(): one pass over the candidate READS of the frontier row (reads never change the model state):
//      the consistent ones are remembered as a bit mask; with eager reads the earliest-invoked consistent read
//      becomes the ONLY child (DESIGN.md: verdict- and witness-preserving);
//   2. next(): every state-changing op in an open slot (write / cas / add / transfer), every consistent read,
//      then the next member of every crashed-op class.
#pragma once
#include <cstdint>

#include "jtb_prep.h"

#if defined(__CUDACC__)
#define JTB_HD __host__ __device__ __forceinline__
#else
#define JTB_HD inline
#endif

namespace jtb {

constexpr uint64_t XKEY_VALID = 1ull << 63;
constexpr uint32_t XRANK_MASK = 0x1fffffffu;

struct I4 {
    int32_t x, y, z, w;
};

JTB_HD I4 ld_i4(const int32_t* p) {
#if defined(__CUDA_ARCH__)
    const int4 v = __ldg(reinterpret_cast<const int4*>(p));
    return I4{v.x, v.y, v.z, v.w};
#else
    return I4{p[0], p[1], p[2], p[3]};
#endif
}
JTB_HD int32_t ld_i32(const int32_t* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
JTB_HD int ld_u8(const uint8_t* p) {
#if defined(__CUDA_ARCH__)
    return (int)__ldg(p);
#else
    return (int)*p;
#endif
}
JTB_HD int ctz64(uint64_t x) {
#if defined(__CUDA_ARCH__)
    return __ffsll((long long)x) - 1;
#else
    return __builtin_ctzll(x);
#endif
}
JTB_HD uint64_t u64_of(int32_t lo, int32_t hi) { return (uint64_t)(uint32_t)lo | ((uint64_t)(uint32_t)hi << 32); }

// What the search shares with the expansion core (device pointers on the device, host vectors in the host walker).
struct ExpandTables {
    const int32_t* rows;
    const ClassRec* classes;
    const int32_t* cls_inv_pos;
    int row_words;
    int sum_off;   // offset of the per-slot summary words in a row (jtb_prep.h); 0 = do not use them
};

template <int KW>
struct Child {
    uint64_t w[KW];
    int cgj;            // frontier rank of the child
    bool done;          // the child linearizes the shard's last :ok op -> the shard is VALID
    int32_t amt, d, c;  // bank: transfer to apply to the parent's balances (amt == 0: none)
};

template <int MODEL, int KW, bool EAGER>
struct Expander {
    static constexpr int SW = MODEL == JTB_MODEL_BANK ? 12 : MODEL == JTB_MODEL_SET ? 8 : 4;  // = slot_words(MODEL)
    static constexpr bool BANK = MODEL == JTB_MODEL_BANK;
    static constexpr bool REG = MODEL == JTB_MODEL_REGISTER || MODEL == JTB_MODEL_CAS_REGISTER;
    static constexpr bool SET = MODEL == JTB_MODEL_SET;

    uint64_t w[KW];
    int32_t bal[8];
    const int32_t* row;
    uint64_t todo, rd_ok;
    int gj, fr_pos, shard, gj_end, cls_base, ncls, rslot, cls_i;
    int32_t reg;

    // loads the frontier row's header; returns the shard id (the caller decides whether the shard is still alive)
    JTB_HD int load_header(const ExpandTables& T) {
        gj = (int)((w[0] >> 32) & XRANK_MASK);
        reg = (int32_t)(uint32_t)w[0];
        row = T.rows + (size_t)gj * T.row_words;
        const I4 h2 = ld_i4(row + 8);
        fr_pos = h2.x; shard = h2.y; gj_end = h2.z; cls_base = h2.w;
        return shard;
    }

    JTB_HD bool read_consistent(const I4& op, const int32_t* cell, uint32_t balhash) const {
        if constexpr (REG) {
            return op.y == JTB_NIL || op.y == reg;
        } else if constexpr (BANK) {
            if ((op.x & OP_HASHED) && (uint32_t)op.z != balhash) return false;
            const I4 lo = ld_i4(cell + 4), hi = ld_i4(cell + 8);
            const int care = op.y;
            bool ok = true;
            ok &= !(care & 1) || bal[0] == lo.x;
            ok &= !(care & 2) || bal[1] == lo.y;
            ok &= !(care & 4) || bal[2] == lo.z;
            ok &= !(care & 8) || bal[3] == lo.w;
            ok &= !(care & 16) || bal[4] == hi.x;
            ok &= !(care & 32) || bal[5] == hi.y;
            ok &= !(care & 64) || bal[6] == hi.z;
            ok &= !(care & 128) || bal[7] == hi.w;
            return ok;
        } else {
            const I4 nc = ld_i4(cell + 4);   // (need, care) u64 pair
            return (w[1] & u64_of(nc.z, nc.w)) == u64_of(nc.x, nc.y);
        }
    }

    // `alive` = the shard is still undecided (a decided shard's configurations produce no children)
    JTB_HD void begin(const ExpandTables& T, bool alive) {
        (void)T;
        const I4 h3 = ld_i4(row + 12);
        const I4 h4 = ld_i4(row + 16);
        ncls = h3.x; rslot = h3.y;
        todo = 0; rd_ok = 0; cls_i = ncls;
        if (!alive) return;
        const uint64_t cand = u64_of(h3.z, h3.w) & ~w[1];
        const uint64_t rdm = u64_of(h4.x, h4.y);
        uint64_t rds = cand & rdm;
        uint32_t balhash = 0;
        if constexpr (BANK) {
            if (rds) {
#pragma unroll
                for (int i = 0; i < 8; ++i) balhash += (uint32_t)bal[i] * bank_hash_c(i);
            }
        }
        // Reads the summary words decide (one contiguous array, all loads independent): only the reads whose summary
        // matches the state are looked at in their cell (bank: exact balances; eager: invocation position).
        if constexpr (!SET) {
            const uint64_t fastm = T.sum_off ? (rds & u64_of(h4.z, h4.w)) : 0ull;
            if (fastm) {
                const int32_t* sum = row + T.sum_off;
                const int32_t want = BANK ? (int32_t)balhash : reg;
                uint64_t match = 0;
                // 16 slots (four 16 B loads, independent) per step: enough loads in flight without a register blow-up
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
                for (int b = 0; b < 4; ++b) {
                    if (!((fastm >> (16 * b)) & 0xffffull)) continue;
                    uint32_t mm = 0;
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const I4 v = ld_i4(sum + 16 * b + 4 * g);
                        uint32_t m4 = (v.x == want) | ((v.y == want) << 1) | ((v.z == want) << 2) | ((v.w == want) << 3);
                        if constexpr (REG)
                            m4 |= (v.x == JTB_NIL) | ((v.y == JTB_NIL) << 1) | ((v.z == JTB_NIL) << 2) | ((v.w == JTB_NIL) << 3);
                        mm |= m4 << (4 * g);
                    }
                    match |= (uint64_t)mm << (16 * b);
                }
                match &= fastm;
                if constexpr (REG && !EAGER) { rd_ok |= match; match = 0; }   // the summary is exact: nothing left to look at
                rds = (rds & ~fastm) | match;
            }
        }
        uint32_t best_inv = 0xffffffffu;
        int best_t = -1;
        while (rds) {
            const int t = ctz64(rds);
            rds &= rds - 1;
            const int32_t* cell = row + ROW_EXTRA + t * SW;
            const I4 op = ld_i4(cell);
            if (!read_consistent(op, cell, balhash)) continue;
            rd_ok |= 1ull << t;
            if (EAGER && (uint32_t)op.w < best_inv) { best_inv = (uint32_t)op.w; best_t = t; }
        }
        if (EAGER && best_t >= 0) {
            rd_ok = todo = 1ull << best_t;   // the earliest-invoked consistent read, exclusively
            return;
        }
        todo = (cand & ~rdm) | rd_ok;
        cls_i = 0;
    }

    // the frontier op is linearized: the frontier passes every return whose op is already linearized
    JTB_HD void advance(const ExpandTables& T, uint64_t& m, int& cgj) const {
        const int32_t* rw = row;
        int adv = 0, k = 0;
        for (;;) {
            const int sl = ld_u8(reinterpret_cast<const uint8_t*>(rw) + k);
            if (sl == 0xff || !((m >> sl) & 1ull)) break;
            m &= ~(1ull << sl);
            ++adv;
            if (++k == 32) { k = 0; rw += (size_t)32 * T.row_words; }
        }
        cgj = gj + 1 + adv;
    }

    JTB_HD int32_t balance_of(int i) const {
        int32_t v = bal[0];
#pragma unroll
        for (int k = 1; k < 8; ++k) v = (i == k) ? bal[k] : v;
        return v;
    }

    // ---- one child at a time, addressable (the level engine hands every child of a warp's 32 configurations to its
    //      own lane; next() below walks the same two lists in order) -----------------------------------------------
    // child that linearizes the op in open slot t (t must be a bit of `todo` as begin() computed it)
    // lazy_op (bank, negative balances allowed): a transfer never fails and the key does not depend on it, so its
    // record is not loaded here; the caller fetches it with load_transfer() only for the children that turn out NEW
    // (ch.d == -1 marks "not loaded")
    JTB_HD bool child_slot(const ExpandTables& T, int t, bool neg_ok, Child<KW>& ch, bool lazy_op = false) const {
        int32_t creg = reg;
        ch.amt = 0; ch.d = 0; ch.c = 0;
        if (!((rd_ok >> t) & 1ull)) {
            if (BANK && lazy_op && neg_ok) {
                ch.d = -1;
            } else {
                const I4 op = ld_i4(row + ROW_EXTRA + t * SW);
                if constexpr (REG) {
                    if ((op.x & 0xff) == JTB_F_WRITE) creg = op.y;
                    else { if (reg != op.y) return false; creg = op.z; }   // cas
                } else if constexpr (BANK) {
                    ch.amt = op.y; ch.d = op.z; ch.c = op.w;
                    if (!neg_ok && balance_of(op.z) - op.y < 0) return false;
                }
            }
        }
#pragma unroll
        for (int i = 0; i < KW; ++i) ch.w[i] = w[i];
        int cgj = gj;
        if (t == rslot) advance(T, ch.w[1], cgj);
        else ch.w[1] |= 1ull << t;
        ch.w[0] = XKEY_VALID | ((uint64_t)(uint32_t)cgj << 32) | (REG ? (uint64_t)(uint32_t)creg : 0ull);
        ch.cgj = cgj;
        ch.done = cgj >= gj_end;
        return true;
    }

    JTB_HD void load_transfer(int t, Child<KW>& ch) const {
        const I4 op = ld_i4(row + ROW_EXTRA + t * SW);
        ch.amt = op.y; ch.d = op.z; ch.c = op.w;
    }

    // child that linearizes the next member of crashed-op class ci of the shard (0 <= ci < ncls)
    JTB_HD bool child_class(const ExpandTables& T, int ci, bool neg_ok, Child<KW>& ch) const {
        const int32_t* q = reinterpret_cast<const int32_t*>(T.classes + cls_base + ci);
        const I4 b = ld_i4(q + 4);   // first, n, word, shift | width << 8
        const int shift = b.w & 0xff, width = b.w >> 8;
        uint64_t field = 0;
#pragma unroll
        for (int i = 1; i < KW; ++i) if (i == b.z) field = w[i];
        const int count = (int)((field >> shift) & ((1ull << width) - 1));
        if (count >= b.y) return false;                                  // the whole class is consumed
        if (ld_i32(T.cls_inv_pos + b.x + count) >= fr_pos) return false;  // its next member is not invoked yet
        const I4 op = ld_i4(q);
        if (op.x & OP_IMPOSSIBLE) return false;
        int32_t creg = reg;
        ch.amt = 0; ch.d = 0; ch.c = 0;
        if constexpr (REG) {
            const int f = op.x & 0xff;
            if (f == JTB_F_WRITE) creg = op.y;
            else if (f == JTB_F_CAS) { if (reg != op.y) return false; creg = op.z; }
            else if (!(op.y == JTB_NIL || op.y == reg)) return false;   // (crashed reads are dropped by the prep)
        } else if constexpr (BANK) {
            if ((op.x & 0xff) != JTB_F_TRANSFER) return false;
            ch.amt = op.y; ch.d = op.z; ch.c = op.w;
            if (!neg_ok && balance_of(op.z) - op.y < 0) return false;
        } else {
            if ((op.x & 0xff) != JTB_F_ADD) return false;
        }
#pragma unroll
        for (int i = 0; i < KW; ++i) ch.w[i] = w[i];
#pragma unroll
        for (int i = 1; i < KW; ++i) if (i == b.z) ch.w[i] += 1ull << shift;
        ch.w[0] = XKEY_VALID | ((uint64_t)(uint32_t)gj << 32) | (REG ? (uint64_t)(uint32_t)creg : 0ull);
        ch.cgj = gj;
        ch.done = false;
        return true;
    }

    JTB_HD bool next(const ExpandTables& T, bool neg_ok, Child<KW>& ch) {
        while (todo) {
            const int t = ctz64(todo);
            todo &= todo - 1;
            if (child_slot(T, t, neg_ok, ch)) return true;
        }
        while (cls_i < ncls) {
            const int ci = cls_i++;
            if (child_class(T, ci, neg_ok, ch)) return true;
        }
        return false;
    }
};

}  // namespace jtb
