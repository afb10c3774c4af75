// jtb_edn_checks.cuh — K19: the host checks of a ledger compose (unexpected-ops, lookup-all-invoked-transfers,
// final-reads, stats) summarised on the device from the bytes of a stored history.edn.
//
// Semantics (include/jtb_check.h, DESIGN.md "K19 stored-history checks"): those of checker.py's UnexpectedOps,
// LookupAllInvokedTransfers, FinalReads and Stats on the op maps edn.read_history makes.  K18's passes 1–5
// (`edn_parse`, ledger-lookups form) read the ops; then, with no thread or warp per op line:
//   - counts and selections over the ops: the client completions by :type, the :fail ops, the :final? :ok reads and
//     lookups (a txn's tag is its first micro-op's), the last client op;
//   - open invokes from K18's (process, position) sort: the last op of a process when it is an invoke, and the first
//     invoke of that run (a max scan), where unexpected-ops' map puts the process;
//   - the invoked ids: every micro-op id of a :t invoke, radix-sorted and made unique (I); one thread per final lookup
//     micro-op finds its id's slot in I, the (lookup, slot) keys are sorted and made unique, and a lookup is suspect
//     when fewer than |I| of them are its own;
//   - final values: one thread per final micro-op checks [keyword int64 map-or-nil] and digests it (128 bits, its
//     position in the op mixed in); a scan sums the digests per op, plus the op's length; the ops of each kind are
//     sorted by digest into classes, and every micro-op is compared with the same-position micro-op of its class's
//     first member, so a collision refuses instead of merging unequal values.
#pragma once
#include "jtb_edn.cuh"

#include <cuda/std/tuple>

namespace jtb {

enum EcErr : uint32_t { EC_MICRO_OP = 1, EC_KEY, EC_VALUE, EC_ID, EC_COLLISION, EC_COUNT };
inline const char* ec_err_text(uint32_t c) {
    static const char* m[EC_COUNT] = {
        "", "a micro-op of a final :ok value that is not [keyword int64-id map-or-nil]",
        "a key in a final :ok value's map other than :debit-acct :credit-acct :amount :debits-posted :credits-posted",
        "a value in a final :ok value's map that is not an int64 or nil", "a transfer invoke's id that is not an int64",
        "a digest collision between unequal final values"};
    return c < EC_COUNT ? m[c] : "unknown refusal";
}

// op->txn-f: the first micro-op's tag; an empty value has none (whatever tag K18 resolved for it)
__device__ __forceinline__ uint8_t ec_tag(const EdnOp& x) { return x.client && x.n_items > 0 ? x.tag : TG_NONE; }

struct EcIsType {   // a client op of this :type
    const EdnOp* op;
    uint8_t type;
    __device__ bool operator()(int32_t o) const { return op[o].client && op[o].type == type; }
};
struct EcIsFinal {   // a :final? :ok op whose first micro-op has this tag
    const EdnOp* op;
    uint8_t tag;
    __device__ bool operator()(int32_t o) const {
        const EdnOp& x = op[o];
        return ec_tag(x) == tag && x.type == JTB_T_OK && (x.flags & JTB_FLAG_FINAL);
    }
};
struct EcIsOpen {   // over the (process, position) order: the last op of its process, and an invoke
    const EdnOp* op;
    const int32_t *cl2, *key2;
    int64_t n;
    __device__ bool operator()(int32_t s) const {
        return (s + 1 == n || key2[s + 1] != key2[s]) && op[cl2[s]].type == JTB_T_INVOKE;
    }
};
struct EcRunStart {   // max-scanned: the start of the run of invokes that ends at s (in the same order)
    const EdnOp* op;
    const int32_t *cl2, *key2;
    __device__ int32_t operator()(int32_t s) const {
        if (op[cl2[s]].type != JTB_T_INVOKE) return s + 1;
        return s == 0 || key2[s - 1] != key2[s] ? s : 0;
    }
};
struct EcMax {
    template <class V>
    __device__ V operator()(V a, V b) const { return a > b ? a : b; }
};
struct EcIsInvokedItem {   // a micro-op of a :t invoke
    const EdnOp* op;
    const EdnItem* it;
    __device__ bool operator()(int32_t k) const {
        const int32_t o = it[k].op;
        return o >= 0 && ec_tag(op[o]) == TG_T && op[o].type == JTB_T_INVOKE;
    }
};
struct EcIsFinalItem {   // a micro-op of a final read or lookup
    const EdnItem* it;
    const int32_t* fin_of;
    __device__ bool operator()(int32_t k) const { return it[k].op >= 0 && fin_of[it[k].op] >= 0; }
};

struct EcDigest {
    uint64_t lo, hi;
};
struct EcAdd {   // lane-wise sum
    __device__ EcDigest operator()(const EcDigest& a, const EcDigest& b) const { return {a.lo + b.lo, a.hi + b.hi}; }
};
struct EcDecomposer {
    __host__ __device__ ::cuda::std::tuple<uint64_t&, uint64_t&> operator()(EcDigest& d) const { return {d.hi, d.lo}; }
};

__device__ __forceinline__ uint64_t ec_fmix(uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    return k ^ (k >> 33);
}
__device__ __forceinline__ void ec_mix(EcDigest& d, uint64_t x) {
    d.lo = ec_fmix(d.lo ^ x);
    d.hi = ec_fmix(d.hi + x * 0x9e3779b97f4a7c15ull + 0x632be59bd9b4e019ull);
}

// the first element of the micro-op at p (its tag, read through a tagged literal) and its end
__device__ __forceinline__ int64_t ec_first(const char* t, int64_t p, int64_t n, int64_t* end) {
    const int64_t q = edn_untag(t, edn_skip_ws(t, p + 1, n), n);
    *end = edn_token_end(t, q, n);
    return q;
}

// one thread per micro-op of a final op (fi[i] = its item): refuses what the digest cannot tell apart, then digests
// it with its position in the op
__global__ void ec_item_kernel(const char* t, int64_t n, const int32_t* fi, int64_t n_fi, const EdnItem* items,
                               const int64_t* it_pos, const EdnOp* op, EcDigest* dig, unsigned long long* err) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_fi) return;
    const int32_t k = fi[i];
    const EdnItem& it = items[k];
    const int64_t p = it_pos[k];
    EcDigest d{0x243f6a8885a308d3ull, 0x13198a2e03707344ull};
    dig[i] = d;
    if (!it.vector || it.n_elems != 3 || it.id_kind != SK_INT || it.map_kind > 1) { edn_fail(err, p, EC_MICRO_OP); return; }
    int64_t e;
    int64_t q = ec_first(t, p, n, &e);
    if (t[q] != ':') { edn_fail(err, p, EC_MICRO_OP); return; }
    uint64_t tag = it.tag;
    if (it.tag == TG_OTHER) {   // any other keyword: its name
        tag = 0xcbf29ce484222325ull;
        for (int64_t x = q + 1; x < e; ++x) tag = (tag ^ (uint8_t)t[x]) * 0x100000001b3ull;
    }
    if (it.map_kind == 1) {   // only the five keys K18 reads, each an int64 or nil
        q = edn_untag(t, edn_skip_ws(t, edn_skip_form(t, q, n), n), n);   // the id
        q = edn_untag(t, edn_skip_ws(t, edn_skip_form(t, q, n), n), n);   // the map
        for (q = q + 1;;) {
            q = edn_skip_ws(t, q, n);
            if (q >= n || t[q] == '}') break;
            if (!(edn_is(t, q, ":debit-acct", 11) || edn_is(t, q, ":credit-acct", 12) || edn_is(t, q, ":amount", 7) ||
                  edn_is(t, q, ":debits-posted", 14) || edn_is(t, q, ":credits-posted", 15))) {
                edn_fail(err, q, EC_KEY);
                return;
            }
            q = edn_skip_form(t, edn_skip_ws(t, edn_skip_form(t, q, n), n), n);   // past the value
        }
        for (int f = 0; f < MV_N; ++f)
            if (it.vk[f] != 0 && it.vk[f] != SK_INT && it.vk[f] != SK_NIL) { edn_fail(err, p, EC_VALUE); return; }
    }
    ec_mix(d, (uint64_t)(k - op[it.op].first_item));
    ec_mix(d, tag);
    ec_mix(d, (uint64_t)it.id);
    ec_mix(d, it.map_kind);
    for (int f = 0; f < MV_N; ++f) {
        ec_mix(d, it.vk[f] == SK_INT ? 2 : it.vk[f] == SK_NIL ? 1 : 0);
        if (it.vk[f] == SK_INT) ec_mix(d, (uint64_t)it.v[f]);
    }
    dig[i] = d;
}

__global__ void ec_fin_of_kernel(const int32_t* fin, int64_t n_fin, int32_t* fin_of) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j < n_fin) fin_of[fin[j]] = (int32_t)j;
}

// index of the first element of sorted a[0, n) that is >= x
template <class V>
__device__ __forceinline__ int64_t ec_lower(const V* a, int64_t n, V x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// each final op's digest: the sum over its micro-ops (an inclusive scan over fi), plus its length
__global__ void ec_op_digest_kernel(const int32_t* fin, int64_t n_fin, const EdnOp* op, const int32_t* fi,
                                    int64_t n_fi, const EcDigest* scan, EcDigest* key, int32_t* val) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n_fin) return;
    const EdnOp& x = op[fin[j]];
    const int64_t b = ec_lower(fi, n_fi, x.first_item), e = b + x.n_items;
    EcDigest d = scan[e - 1];
    if (b > 0) d = {d.lo - scan[b - 1].lo, d.hi - scan[b - 1].hi};
    key[j] = {d.lo + (uint64_t)x.n_items, d.hi + (uint64_t)x.n_items};
    val[j] = (int32_t)j;
}

struct EcHead {   // 1 at the first op of a class (sorted by digest)
    const EcDigest* key;
    __device__ int32_t operator()(int32_t s) const {
        return s == 0 || key[s].lo != key[s - 1].lo || key[s].hi != key[s - 1].hi;
    }
};
struct EcHeadPos {
    EcHead head;
    __device__ int32_t operator()(int32_t s) const { return head(s) ? s : 0; }
};

// sorted position s of one kind's final ops (val: their indices in fin): its op's class and the op that represents
// the class (its first member in the sort)
__global__ void ec_class_kernel(const int32_t* val, const int32_t* csum, const int32_t* hpos, int64_t n, int32_t* cls,
                                int32_t* rep) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    cls[val[s]] = csum[s] - 1;
    rep[val[s]] = val[hpos[s]];
}

__device__ __forceinline__ bool ec_same_tag(const char* t, int64_t n, const EdnItem& a, int64_t pa, const EdnItem& b,
                                            int64_t pb) {
    if (a.tag != b.tag) return false;
    if (a.tag != TG_OTHER) return true;
    int64_t ea, eb;
    const int64_t qa = ec_first(t, pa, n, &ea), qb = ec_first(t, pb, n, &eb);
    if (ea - qa != eb - qb) return false;
    for (int64_t x = 0; x < ea - qa; ++x)
        if (t[qa + x] != t[qb + x]) return false;
    return true;
}

// every final micro-op against the same-position micro-op of its class's representative
__global__ void ec_confirm_kernel(const char* t, int64_t n, const int32_t* fi, int64_t n_fi, const EdnItem* items,
                                  const int64_t* it_pos, const EdnOp* op, const int64_t* ops, const int32_t* fin,
                                  const int32_t* fin_of, const int32_t* rep, unsigned long long* err) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_fi) return;
    const int32_t k = fi[i];
    const EdnItem& a = items[k];
    const int32_t o = a.op, r = fin[rep[fin_of[o]]];
    if (r == o) return;
    if (op[r].n_items != op[o].n_items) { edn_fail(err, ops[o], EC_COLLISION); return; }
    const int32_t k2 = op[r].first_item + (k - op[o].first_item);
    const EdnItem& b = items[k2];
    bool same = ec_same_tag(t, n, a, it_pos[k], b, it_pos[k2]) && a.id == b.id && a.map_kind == b.map_kind;
    for (int f = 0; f < MV_N && same; ++f)
        same = a.vk[f] == b.vk[f] && (a.vk[f] != SK_INT || a.v[f] == b.v[f]);
    if (!same) edn_fail(err, ops[o], EC_COLLISION);
}

// the ids of the :t invokes' micro-ops (ii: their items)
__global__ void ec_invoked_kernel(const int32_t* ii, int64_t n_ii, const EdnItem* items, const int64_t* it_pos,
                                  int64_t* ids, unsigned long long* err) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_ii) return;
    const EdnItem& it = items[ii[i]];
    if (it.id_kind != SK_INT) edn_fail(err, it_pos[ii[i]], EC_ID);
    ids[i] = it.id;
}

// a final lookup's micro-op: (lookup ordinal << 32 | the slot of its id in I); ~0 for a read's or an id not in I
__global__ void ec_slot_kernel(const int32_t* fi, int64_t n_fi, const EdnItem* items, const int32_t* fin_of,
                               int64_t n_fr, const int64_t* inv, int64_t n_inv, uint64_t* key) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_fi) return;
    const EdnItem& it = items[fi[i]];
    const int64_t j = fin_of[it.op] - n_fr;
    uint64_t w = ~0ull;
    if (j >= 0) {
        const int64_t s = ec_lower(inv, n_inv, it.id);
        if (s < n_inv && inv[s] == it.id) w = ((uint64_t)j << 32) | (uint64_t)s;
    }
    key[i] = w;
}

// a final lookup is suspect when fewer than |I| distinct (lookup, slot) keys are its own
__global__ void ec_suspect_kernel(const uint64_t* uk, int64_t n_uk, int64_t n_fl, int64_t n_inv, uint8_t* suspect) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n_fl) return;
    const int64_t a = ec_lower(uk, n_uk, (uint64_t)j << 32), b = ec_lower(uk, n_uk, (uint64_t)(j + 1) << 32);
    suspect[j] = b - a < n_inv;
}

// the op's '{' and the position after its matching '}' (the brackets sorted by (level, position) pair up)
__device__ __forceinline__ int64_t ec_map_end(const uint32_t* lv2, const int64_t* br2, int64_t nb, uint32_t level,
                                              int64_t pos) {
    int64_t lo = 0, hi = nb / 2;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        const uint32_t l = lv2[2 * mid];
        if (l < level || (l == level && br2[2 * mid] < pos)) lo = mid + 1;
        else hi = mid;
    }
    return br2[2 * lo + 1] + 1;
}

// the flagged ops' records: list[i] is an op, or (via) a position in the (process, position) order
struct EcRecordIn {
    const int32_t* list;
    int64_t n;
    const int32_t* via;         // may be null
    const int32_t* run_start;   // open invokes: per position, the start of its run of invokes; may be null
    const int32_t* cls;         // may be null
    const uint8_t* suspect;     // may be null
};
__global__ void ec_record_kernel(EcRecordIn in, const int64_t* ops, const EdnOp* op, const int32_t* field,
                                 const uint32_t* lv2, const int64_t* br2, int64_t nb, uint32_t level,
                                 jtb_edn_flag* out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= in.n) return;
    const int32_t s = in.list[i], o = in.via ? in.via[s] : s;
    const EdnOp& x = op[o];
    jtb_edn_flag r{};
    r.op = o;
    r.begin = ops[o];
    r.end = ec_map_end(lv2, br2, nb, level, ops[o]);
    r.has_time = field[(int64_t)o * EK_N + EK_TIME] != 0;
    r.has_index = field[(int64_t)o * EK_N + EK_INDEX] != 0;
    r.time = r.has_time ? x.time : 0;
    r.index = r.has_index ? x.index : 0;
    r.first = in.run_start ? in.via[in.run_start[s]] : -1;
    r.cls = in.cls ? in.cls[i] : -1;
    r.suspect = in.suspect ? in.suspect[i] : 0;
    out[i] = r;
}

// frees the page-locked arrays of out and clears it
inline void jtb_edn_checks_release(jtb_edn_checks* out) {
    for (void* p : {(void*)out->open, (void*)out->fails, (void*)out->final_reads, (void*)out->final_lookups})
        if (p) cudaFreeHost(p);
    std::memset(out, 0, sizeof *out);
}

// the host side of jtb_ledger_edn_checks
inline int run_ledger_edn_checks(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const char* text, int64_t n,
                                 int32_t flags, jtb_edn_checks* out, std::string& err) {
    using Clock = std::chrono::steady_clock;
    const auto t0 = Clock::now();
    if (!out || n < 0 || (n > 0 && !text)) return input_error(err, "malformed arguments");
    if (flags != 0) return input_error(err, "flags must be 0");
    std::memset(out, 0, sizeof *out);
    out->last.op = -1;
    const int T = 256;
    CallAllocs A;
    EdnParse P(st, A);
    EdnRefusal r;
    auto refuse = [&](const EdnRefusal& why) {
        out->refused = 1;
        out->refused_at = why.at;
        std::snprintf(out->refused_reason, sizeof out->refused_reason, "%s", why.reason);
        out->seconds_h2d = std::chrono::duration<double>(P.t_h2d - t0).count();
        out->seconds_total = std::chrono::duration<double>(Clock::now() - t0).count();
        return 0;
    };
    if (edn_parse(P, ev0, text, n, JTB_FORM_LEDGER_LOOKUPS, r, err) != 0) return -1;
    if (r.reason) return refuse(r);
    size_t& bytes = P.bytes;
    const int64_t n_ops = P.n_ops, n_it = P.n_it, n_cl = P.n_cl;
    const EdnOp* op = P.op;
    const EdnItem* items = P.items;
    unsigned long long* d_err = P.err;   // K18 found nothing: the word is free for this call's refusals
    auto oi = thrust::counting_iterator<int32_t>(0);
    auto ec_error = [&](bool* refused) -> int {
        unsigned long long w = ~0ull;
        JTB_OK(P.error_word(&w));
        if (w != ~0ull) {
            r.at = (int64_t)(w >> 8);
            r.reason = ec_err_text((uint32_t)(w & 0xff));
            *refused = true;
        }
        return 0;
    };
    auto list = [&](auto in, int64_t n_in, auto pred, int32_t** outp, int64_t* n_out) -> cudaError_t {
        cudaError_t e = P.count(in, n_in, pred, n_out);
        if (e == cudaSuccess) e = A.alloc(outp, (size_t)*n_out);
        return e == cudaSuccess && *n_out ? P.select_into(in, n_in, pred, *outp) : e;
    };

    // ---- counts, fails, final ops -------------------------------------------------------------------------------------
    int32_t *fails, *fin, *fi, *fin_of, *ii;
    int64_t n_fail = 0, n_fr = 0, n_fl = 0, n_fi = 0, n_ii = 0;
    JTB_OK(P.count(oi, n_ops, EcIsType{op, JTB_T_OK}, &out->n_ok));
    JTB_OK(P.count(oi, n_ops, EcIsType{op, JTB_T_INFO}, &out->n_info));
    JTB_OK(list(oi, n_ops, EcIsType{op, JTB_T_FAIL}, &fails, &n_fail));
    JTB_OK(P.count(oi, n_ops, EcIsFinal{op, TG_R}, &n_fr));
    JTB_OK(P.count(oi, n_ops, EcIsFinal{op, TG_LT}, &n_fl));
    JTB_OK(A.alloc(&fin, (size_t)(n_fr + n_fl)));   // the final reads, then the final lookups
    if (n_fr) JTB_OK(P.select_into(oi, n_ops, EcIsFinal{op, TG_R}, fin));
    if (n_fl) JTB_OK(P.select_into(oi, n_ops, EcIsFinal{op, TG_LT}, fin + n_fr));
    const int64_t n_fin = n_fr + n_fl;
    JTB_OK(A.alloc(&fin_of, (size_t)n_ops));
    JTB_OK(cudaMemsetAsync(fin_of, 0xff, (size_t)n_ops * 4, st));
    if (n_fin) ec_fin_of_kernel<<<edn_blocks(n_fin), T, 0, st>>>(fin, n_fin, fin_of);
    JTB_OK(cudaGetLastError());
    JTB_OK(list(oi, n_it, EcIsFinalItem{items, fin_of}, &fi, &n_fi));
    JTB_OK(list(oi, n_it, EcIsInvokedItem{op, items}, &ii, &n_ii));

    // ---- open invokes -------------------------------------------------------------------------------------------------
    int32_t *open = nullptr, *run_start = nullptr;
    int64_t n_open = 0;
    if (n_cl) {
        JTB_OK(list(oi, n_cl, EcIsOpen{op, P.cl2, P.key2, n_cl}, &open, &n_open));
        JTB_OK(A.alloc(&run_start, (size_t)n_cl));
        auto rs = thrust::make_transform_iterator(oi, EcRunStart{op, P.cl2, P.key2});
        JTB_OK(cub::DeviceScan::InclusiveScan(nullptr, bytes, rs, run_start, EcMax{}, n_cl, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceScan::InclusiveScan(P.tmp, bytes, rs, run_start, EcMax{}, n_cl, st));
    }

    // ---- the invoked ids I, and the final micro-ops' checks and digests ---------------------------------------------
    int64_t *ids, *ids2, *inv, n_inv = 0;
    JTB_OK(A.alloc(&ids, (size_t)n_ii));
    JTB_OK(A.alloc(&ids2, (size_t)n_ii));
    JTB_OK(A.alloc(&inv, (size_t)n_ii));
    EcDigest *dig, *dscan;
    JTB_OK(A.alloc(&dig, (size_t)n_fi));
    JTB_OK(A.alloc(&dscan, (size_t)n_fi));
    if (n_ii) {
        ec_invoked_kernel<<<edn_blocks(n_ii), T, 0, st>>>(ii, n_ii, items, P.it_pos, ids, d_err);
        JTB_OK(cudaGetLastError());
        JTB_OK(cub::DeviceRadixSort::SortKeys(nullptr, bytes, ids, ids2, n_ii, 0, 64, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceRadixSort::SortKeys(P.tmp, bytes, ids, ids2, n_ii, 0, 64, st));
        JTB_OK(cub::DeviceSelect::Unique(nullptr, bytes, ids2, inv, P.d_cnt, n_ii, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceSelect::Unique(P.tmp, bytes, ids2, inv, P.d_cnt, n_ii, st));
        JTB_OK(P.fetch(&n_inv, P.d_cnt));
    }
    if (n_fi) {
        ec_item_kernel<<<edn_blocks(n_fi), T, 0, st>>>(P.text, P.N, fi, n_fi, items, P.it_pos, op, dig, d_err);
        JTB_OK(cudaGetLastError());
    }
    bool refused = false;
    if (ec_error(&refused) != 0) return -1;
    if (refused) return refuse(r);

    // ---- suspect lookups ----------------------------------------------------------------------------------------------
    uint8_t* suspect;
    JTB_OK(A.alloc(&suspect, (size_t)n_fl));
    if (n_fl) {
        uint64_t *sk, *sk2, *uk;
        int64_t n_uk = 0;
        JTB_OK(A.alloc(&sk, (size_t)n_fi));
        JTB_OK(A.alloc(&sk2, (size_t)n_fi));
        JTB_OK(A.alloc(&uk, (size_t)n_fi));
        ec_slot_kernel<<<edn_blocks(n_fi), T, 0, st>>>(fi, n_fi, items, fin_of, n_fr, inv, n_inv, sk);
        JTB_OK(cudaGetLastError());
        int end_bit = 33;   // the slot's 32 bits and the lookup ordinal's; ~0 stays last
        while (end_bit < 64 && (n_fl >> (end_bit - 32))) ++end_bit;
        JTB_OK(cub::DeviceRadixSort::SortKeys(nullptr, bytes, sk, sk2, n_fi, 0, end_bit, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceRadixSort::SortKeys(P.tmp, bytes, sk, sk2, n_fi, 0, end_bit, st));
        JTB_OK(cub::DeviceSelect::Unique(nullptr, bytes, sk2, uk, P.d_cnt, n_fi, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceSelect::Unique(P.tmp, bytes, sk2, uk, P.d_cnt, n_fi, st));
        JTB_OK(P.fetch(&n_uk, P.d_cnt));
        ec_suspect_kernel<<<edn_blocks(n_fl), T, 0, st>>>(uk, n_uk, n_fl, n_inv, suspect);
        JTB_OK(cudaGetLastError());
    }

    // ---- classes of equal final values, then their exact confirmation -------------------------------------------------
    int32_t *cls, *rep;
    JTB_OK(A.alloc(&cls, (size_t)n_fin));
    JTB_OK(A.alloc(&rep, (size_t)n_fin));
    int64_t n_classes[2] = {0, 0};
    if (n_fin) {
        EcDigest *key, *key2;
        int32_t *val, *val2, *csum, *hpos;
        JTB_OK(A.alloc(&key, (size_t)n_fin));
        JTB_OK(A.alloc(&key2, (size_t)n_fin));
        JTB_OK(A.alloc(&val, (size_t)n_fin));
        JTB_OK(A.alloc(&val2, (size_t)n_fin));
        JTB_OK(A.alloc(&csum, (size_t)n_fin));
        JTB_OK(A.alloc(&hpos, (size_t)n_fin));
        JTB_OK(cub::DeviceScan::InclusiveScan(nullptr, bytes, dig, dscan, EcAdd{}, n_fi, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceScan::InclusiveScan(P.tmp, bytes, dig, dscan, EcAdd{}, n_fi, st));
        ec_op_digest_kernel<<<edn_blocks(n_fin), T, 0, st>>>(fin, n_fin, op, fi, n_fi, dscan, key, val);
        JTB_OK(cudaGetLastError());
        const int64_t range[3] = {0, n_fr, n_fin};   // the reads' classes, then the lookups'
        for (int kind = 0; kind < 2; ++kind) {
            const int64_t j0 = range[kind], m = range[kind + 1] - j0;
            if (!m) continue;
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, key + j0, key2 + j0, val + j0, val2 + j0, m,
                                                   EcDecomposer{}, st));
            JTB_OK(P.need_tmp(bytes));
            JTB_OK(cub::DeviceRadixSort::SortPairs(P.tmp, bytes, key + j0, key2 + j0, val + j0, val2 + j0, m,
                                                   EcDecomposer{}, st));
            auto heads = thrust::make_transform_iterator(oi, EcHead{key2 + j0});
            auto hp = thrust::make_transform_iterator(oi, EcHeadPos{EcHead{key2 + j0}});
            JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, bytes, heads, csum + j0, m, st));
            JTB_OK(P.need_tmp(bytes));
            JTB_OK(cub::DeviceScan::InclusiveSum(P.tmp, bytes, heads, csum + j0, m, st));
            JTB_OK(cub::DeviceScan::InclusiveScan(nullptr, bytes, hp, hpos + j0, EcMax{}, m, st));
            JTB_OK(P.need_tmp(bytes));
            JTB_OK(cub::DeviceScan::InclusiveScan(P.tmp, bytes, hp, hpos + j0, EcMax{}, m, st));
            ec_class_kernel<<<edn_blocks(m), T, 0, st>>>(val2 + j0, csum + j0, hpos + j0, m, cls, rep);
            JTB_OK(cudaGetLastError());
            int32_t last = 0;
            JTB_OK(cudaMemcpyAsync(&last, csum + j0 + m - 1, 4, cudaMemcpyDeviceToHost, st));
            JTB_OK(cudaStreamSynchronize(st));
            n_classes[kind] = last;
        }
        ec_confirm_kernel<<<edn_blocks(n_fi), T, 0, st>>>(P.text, P.N, fi, n_fi, items, P.it_pos, op, P.ops, fin,
                                                          fin_of, rep, d_err);
        JTB_OK(cudaGetLastError());
        if (ec_error(&refused) != 0) return -1;
        if (refused) return refuse(r);
    }

    // ---- the flagged ops' records ---------------------------------------------------------------------------------------
    jtb_edn_flag *d_open, *d_fails, *d_fin, *d_last;
    JTB_OK(A.alloc(&d_open, (size_t)n_open));
    JTB_OK(A.alloc(&d_fails, (size_t)n_fail));
    JTB_OK(A.alloc(&d_fin, (size_t)n_fin));
    JTB_OK(A.alloc(&d_last, 1));
    const uint32_t level = (uint32_t)P.base + 1;   // the level of an op map's brackets
    auto record = [&](EcRecordIn in, jtb_edn_flag* dst) -> cudaError_t {
        if (!in.n) return cudaSuccess;
        ec_record_kernel<<<edn_blocks(in.n), T, 0, st>>>(in, P.ops, op, P.field, P.lv2, P.br2, P.nb, level, dst);
        return cudaGetLastError();
    };
    JTB_OK(record({open, n_open, P.cl2, run_start, nullptr, nullptr}, d_open));
    JTB_OK(record({fails, n_fail, nullptr, nullptr, nullptr, nullptr}, d_fails));
    JTB_OK(record({fin, n_fr, nullptr, nullptr, cls, nullptr}, d_fin));
    JTB_OK(record({fin + n_fr, n_fl, nullptr, nullptr, cls + n_fr, suspect}, d_fin + n_fr));
    if (n_cl) JTB_OK(record({P.cl + n_cl - 1, 1, nullptr, nullptr, nullptr, nullptr}, d_last));
    JTB_OK(cudaEventRecord(ev1, st));
    JTB_OK(cudaStreamSynchronize(st));
    const auto t2 = Clock::now();
    float ms = 0;
    JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));

    // ---- copied into page-locked host memory the library owns -----------------------------------------------------------
    const size_t F = sizeof(jtb_edn_flag);
    out->open = (jtb_edn_flag*)jtb_host_alloc(n_open * F);
    out->fails = (jtb_edn_flag*)jtb_host_alloc(n_fail * F);
    out->final_reads = (jtb_edn_flag*)jtb_host_alloc(n_fr * F);
    out->final_lookups = (jtb_edn_flag*)jtb_host_alloc(n_fl * F);
    if (!out->open || !out->fails || !out->final_reads || !out->final_lookups) {
        jtb_edn_checks_release(out);
        return input_error(err, "jtb_host_alloc failed for the flagged ops");
    }
    cudaError_t ce = cudaSuccess;
    for (auto [dst, src, m] : {std::tuple<void*, const void*, int64_t>{out->open, d_open, n_open},
                               {out->fails, d_fails, n_fail}, {out->final_reads, d_fin, n_fr},
                               {out->final_lookups, d_fin + n_fr, n_fl}, {&out->last, d_last, n_cl ? 1 : 0}})
        if (ce == cudaSuccess && m) ce = cudaMemcpyAsync(dst, src, m * F, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) {
        jtb_edn_checks_release(out);
        err = std::string("copying the flagged ops back: ") + cudaGetErrorString(ce);
        return -1;
    }
    out->n_ops = n_ops;
    out->n_client = n_cl;
    out->n_fail = n_fail;
    out->n_open = n_open;
    out->n_final_reads = n_fr;
    out->n_final_lookups = n_fl;
    out->n_read_classes = n_classes[0];
    out->n_lookup_classes = n_classes[1];
    out->n_invoked = n_inv;
    for (int64_t j = 0; j < n_fl; ++j) out->n_suspect += out->final_lookups[j].suspect;
    const auto t3 = Clock::now();
    out->seconds_h2d = std::chrono::duration<double>(P.t_h2d - t0).count();
    out->seconds_kernel = ms * 1e-3;
    out->seconds_d2h = std::chrono::duration<double>(t3 - t2).count();
    out->seconds_total = std::chrono::duration<double>(t3 - t0).count();
    return 0;
}
}  // namespace jtb
