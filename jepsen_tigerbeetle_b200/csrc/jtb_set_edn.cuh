// jtb_set_edn.cuh — K20: a stored set-full history.edn read on the device into the keyed "set" form.
//
// Semantics (include/jtb_check.h, DESIGN.md "K20 stored set-history reader"): the arrays are exactly those of
// `edn.read_history(text, independent=True)` followed by `history.flatten_ops(ops, "set")`, one CSR shard per key;
// where that Python path raises, the call returns rc < 0.  The EDN subset and the op fields (:type, :time, :process,
// :index, :final?) are K18's (jtb_edn.cuh, passes 1–4 of `edn_parse_forms`).
//
// After those passes, with form starts selected one level deeper (a member of `[k #{…}]` sits at base + 3):
//   5. one thread per op reads :f and the kind of its :value; one thread per form at base + 2 counts the elements of
//      each op's :value, so a 2-element vector or list is a jepsen.independent tuple [key value]; one thread per op then
//      reads the key and the add value, or where a read's members are (the value's elements, or the tuple's second
//      element's), and whether they are a set (sorted) or a vector or list (kept in order).
//   6. one thread per candidate member (every form at base + 2 and base + 3) keeps the members of the reads and checks
//      them; the payload length of each read is their count.
//   7. the kept events are split into keyed and unkeyed ones; the keyed ones go through the stable key partition of
//      jtb_partition.cuh on device-resident keys, and the unkeyed ones follow in history order as the last shard (key id
//      -1), as `(k is None, k)` orders them.  Payload offsets come from a cub scan over the partitioned events.
//   8. the members are radix-sorted by (partitioned event, member) for sets and by partitioned event alone for vectors
//      (the sort is stable, so vectors keep their order): the sorted values are the payload.  A set literal with a
//      repeated member is refused (edn.py would drop the repeat).
#pragma once
#include "jtb_edn.cuh"
#include "jtb_partition.cuh"

namespace jtb {

// the set reader's refusals, after K18's codes (the error word keeps the code in its low 8 bits)
enum SetEdnErr : uint32_t {
    SE_F = EE_COUNT, SE_KEY, SE_KEY_INT64, SE_ADD, SE_READ, SE_MEMBER, SE_REPEAT, SE_END
};
inline const char* set_edn_err_text(uint32_t c) {
    static const char* m[SE_END - EE_COUNT] = {
        ":f other than :add or :read", "a key that is not an integer or nil", "a key outside int64",
        "an add value that is not an integer or nil", "a read value that is not nil, a vector, a list or a set",
        "a read member that is not an integer", "a set literal with a repeated member"};
    return c >= EE_COUNT && c < SE_END ? m[c - EE_COUNT] : edn_err_text(c);
}

// a form's kind: SV_* for a collection or a string, else edn_scalar's SK_*
enum : uint8_t { SV_SEQ = 16, SV_SET, SV_MAP, SV_STR };
// what a read's members are: none (nil), the :value's elements, or the elements of the tuple's second element
enum : uint8_t { MS_NONE = 0, MS_VALUE, MS_TUPLE };

struct SetOp : EdnOp {
    int64_t key;       // the event's key when keyed
    uint8_t keyed;     // 0: the key is nil or the value is not a tuple (the last shard, key id -1)
    uint8_t msrc;      // MS_*
    uint8_t sorted;    // the members are a set literal
};

// the kind of the form starting at p (and, for SK_INT, its value in *v)
__device__ __forceinline__ uint8_t set_form_kind(const char* t, int64_t p, int64_t n, int64_t* v) {
    p = edn_untag(t, p, n);
    if (p >= n) return SK_OTHER;
    const char c = t[p];
    const bool hash = p > 0 && t[p - 1] == '#';
    if (c == '[' || c == '(') return hash ? SK_OTHER : SV_SEQ;   // #[ is not EDN
    if (c == '{') return hash ? SV_SET : SV_MAP;
    if (c == '"') return SV_STR;
    return edn_scalar(t, p, n, v);
}

// the int32 of an add value or a member, or the reason it is refused
__device__ __forceinline__ uint32_t set_i32_error(uint8_t kind, int64_t v, uint32_t other) {
    if (kind == SK_INT) return v >= INT_MIN && v <= INT_MAX ? 0u : (uint32_t)EE_INT32;
    return kind == SK_BIG ? (uint32_t)EE_INT32 : kind == SK_BADNUM ? (uint32_t)EE_NUMBER : other;
}

// ---- 5: op fields, :value elements, keys and read kinds --------------------------------------------------------------
__global__ void set_op_kernel(const char* t, int64_t n, const int64_t* ops, int64_t n_ops, const int64_t* ch,
                              const int32_t* n_child, const int32_t* field, SetOp* out, unsigned long long* err) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= n_ops) return;
    SetOp op{};
    op.value_child = -1;
    op.first_item = INT_MAX;
    op.plen = -1;
    op.vkind = SK_NIL;
    const int32_t* fo = field + o * EK_N;
    if (edn_op_fields(t, n, o, ops[o], ch, n_child, fo, op, err) && op.client) {
        const int64_t pf = fo[EK_F] ? ch[fo[EK_F] - 1] : ops[o];
        if (fo[EK_F] && edn_is(t, pf, ":add", 4)) {
            op.f = JTB_F_ADD;
        } else if (fo[EK_F] && edn_is(t, pf, ":read", 5)) {
            op.f = JTB_F_READ;
        } else {
            edn_fail(err, pf, SE_F);
            op.client = 0;   // refused: no later pass reads it
        }
        if (op.client && fo[EK_VALUE]) {
            int64_t v = 0;
            op.value_child = fo[EK_VALUE] - 1;
            op.vkind = set_form_kind(t, ch[op.value_child], n, &v);
        }
    }
    out[o] = op;
}

// one thread per form at base + 2: the elements of a client op's :value (contiguous in it_pos)
__global__ void set_item_kernel(const int64_t* ops, int64_t n_ops, const int64_t* ch, int64_t n_ch,
                                const int64_t* it_pos, int64_t n_it, SetOp* op) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_it) return;
    const int64_t pos = it_pos[k];
    const int64_t o = edn_floor(ops, n_ops, pos);
    if (o < 0 || !op[o].client || op[o].value_child < 0 || edn_floor(ch, n_ch, pos) != op[o].value_child) return;
    atomicMin(&op[o].first_item, (int32_t)k);
    atomicAdd(&op[o].n_items, 1);
}

// what each client op becomes: its key (a 2-element vector or list is [key value]), an add's value (nil: dropped), or
// where a read's members are
__global__ void set_event_kernel(const char* t, int64_t n, int64_t n_ops, const int64_t* ch, const int64_t* it_pos,
                                 SetOp* op, unsigned long long* err) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= n_ops) return;
    SetOp& x = op[o];
    x.keep = 0;
    if (!x.client) return;
    const bool tuple = x.vkind == SV_SEQ && x.n_items == 2;
    const int64_t vpos = tuple ? it_pos[x.first_item + 1] : x.value_child >= 0 ? ch[x.value_child] : -1;
    int64_t v = 0;
    const uint8_t vk = vpos >= 0 ? set_form_kind(t, vpos, n, &v) : (uint8_t)SK_NIL;
    if (x.f == JTB_F_ADD) {
        if (vk == SK_NIL) return;   // the [nil nil] add-ok of a rejected account: no event, and its key is not read
        const uint32_t e = set_i32_error(vk, v, SE_ADD);
        if (e) edn_fail(err, vpos, e);
        else x.a = (int32_t)v;
    } else if (vk == SV_SEQ || vk == SV_SET) {
        x.plen = 0;   // the member pass counts them
        x.msrc = tuple ? MS_TUPLE : MS_VALUE;
        x.sorted = vk == SV_SET;
    } else if (vk != SK_NIL) {
        edn_fail(err, vpos, vk == SK_BADNUM ? (uint32_t)EE_NUMBER : (uint32_t)SE_READ);
    }
    x.keep = 1;
    if (tuple) {
        const int64_t kp = it_pos[x.first_item];
        int64_t k = 0;
        const uint8_t kk = set_form_kind(t, kp, n, &k);
        if (kk == SK_INT) {
            x.keyed = 1;
            x.key = k;
        } else if (kk != SK_NIL) {
            edn_fail(err, kp, kk == SK_BIG ? (uint32_t)SE_KEY_INT64 : kk == SK_BADNUM ? (uint32_t)EE_NUMBER
                                                                                      : (uint32_t)SE_KEY);
        }
    }
}

// ---- 6: members -----------------------------------------------------------------------------------------------------
// One thread per candidate k: the forms at base + 2 (k < n_it) and then those at base + 3.  mop[k]: the op whose read
// k is a member of, -1 none; mval[k]: the member.
__global__ void set_member_kernel(const char* t, int64_t n, const int64_t* ops, int64_t n_ops, const int64_t* it_pos,
                                  int64_t n_it, const int64_t* deep, int64_t n_deep, SetOp* op, int32_t* mop,
                                  int32_t* mval, unsigned long long* err) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_it + n_deep) return;
    const bool item = k < n_it;
    const int64_t pos = item ? it_pos[k] : deep[k - n_it];
    int32_t o = (int32_t)edn_floor(ops, n_ops, pos);
    if (o >= 0) {
        const SetOp& x = op[o];
        if (!x.keep || x.msrc != (item ? MS_VALUE : MS_TUPLE)) o = -1;
        else if (item && (k < x.first_item || k >= (int64_t)x.first_item + x.n_items)) o = -1;
        // a form at base + 3 lies in the base + 2 form that starts last before it
        else if (!item && edn_floor(it_pos, n_it, pos) != (int64_t)x.first_item + 1) o = -1;
    }
    mop[k] = o;
    mval[k] = 0;
    if (o < 0) return;
    int64_t v = 0;
    const uint32_t e = set_i32_error(set_form_kind(t, pos, n, &v), v, SE_MEMBER);
    if (e) edn_fail(err, pos, e);
    else mval[k] = (int32_t)v;
    atomicAdd((unsigned long long*)&op[o].plen, 1ull);
}

// ---- 7: events and the key partition --------------------------------------------------------------------------------
struct SetKept {   // kept events with (want = 1) or without (want = 0) a key
    const SetOp* op;
    uint8_t want;
    __device__ bool operator()(int32_t o) const { return op[o].keep && op[o].keyed == want; }
};

__global__ void set_key_kernel(const SetOp* op, const int32_t* keyed, int64_t n, int64_t* key) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) key[i] = op[keyed[i]].key;
}

// sop[s]: the op of partitioned event s (the keyed events in partition order, then the unkeyed ones); spos[op] = s
__global__ void set_order_kernel(const int32_t* keyed, const int32_t* order, int64_t n_keyed, const int32_t* unkeyed,
                                 int64_t n_events, int32_t* sop, int32_t* spos) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_events) return;
    const int32_t o = s < n_keyed ? keyed[order[s]] : unkeyed[s - n_keyed];
    sop[s] = o;
    spos[o] = (int32_t)s;
}

struct SetPlen {
    const SetOp* op;
    const int32_t* sop;
    __device__ int64_t operator()(int64_t s) const { return max(op[sop[s]].plen, (int64_t)0); }
};

__global__ void set_write_events_kernel(const SetOp* op, const int32_t* sop, int64_t n_events, const int64_t* poff_incl,
                                        EdnEvents e) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_events) return;
    const SetOp& x = op[sop[s]];
    e.type[s] = x.type;
    e.f[s] = x.f;
    e.flags[s] = x.flags;
    e.process[s] = x.process;
    e.index[s] = x.index;
    e.time_ns[s] = x.time;
    e.a[s] = x.a;
    e.b[s] = 0;
    e.c[s] = 0;
    e.payload_off[s] = poff_incl[s] - max(x.plen, (int64_t)0);
    e.payload_len[s] = (int32_t)x.plen;
}

// ---- 8: the payload -------------------------------------------------------------------------------------------------
// the sort key of candidate k: (partitioned event << 32) | (member ^ sign bit) for a set, | 0 for a vector or list;
// all ones for a candidate that is not a member (it sorts last: the events fit below the sort's top bits)
__global__ void set_sort_key_kernel(const int32_t* mop, const int32_t* mval, int64_t n_m, const SetOp* op,
                                    const int32_t* spos, uint64_t* key) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_m) return;
    const int32_t o = mop[k];
    if (o < 0) { key[k] = ~0ull; return; }
    const uint32_t low = op[o].sorted ? (uint32_t)mval[k] ^ 0x80000000u : 0u;
    key[k] = ((uint64_t)(uint32_t)spos[o] << 32) | low;
}

// a set literal's members, sorted: a repeat is refused (edn.py keeps one, Clojure's reader rejects the literal)
__global__ void set_repeat_kernel(const uint64_t* key, int64_t n_payload, const SetOp* op, const int32_t* sop,
                                  const int64_t* ops, unsigned long long* err) {
    const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (m == 0 || m >= n_payload || key[m] != key[m - 1]) return;
    const int32_t o = sop[key[m] >> 32];
    if (op[o].sorted) edn_fail(err, ops[o], SE_REPEAT);
}

// the host side of jtb_read_set_edn
inline int run_read_set_edn(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const char* text, int64_t n,
                            int32_t flags, jtb_edn_history* out, std::string& err) {
    using Clock = std::chrono::steady_clock;
    const auto t0 = Clock::now();
    if (!out || n < 0 || (n > 0 && !text)) return input_error(err, "malformed arguments");
    if (flags != 0) return input_error(err, "flags must be 0");
    std::memset(out, 0, sizeof *out);
    const int T = 256;
    CallAllocs A;
    EdnParse P(st, A);
    EdnRefusal r;
    unsigned long long w = ~0ull;
    auto refuse = [&]() {
        if (r.at >= 0) return input_error(err, "history.edn at byte %lld: %s", (long long)r.at, r.reason);
        return input_error(err, "history.edn: %s", r.reason);
    };
    auto refused_word = [&]() {   // the first refusal in the file, if any
        if (w == ~0ull) return false;
        r.at = (int64_t)(w >> 8);
        r.reason = set_edn_err_text((uint32_t)(w & 0xff));
        return true;
    };
    if (edn_parse_forms(P, ev0, text, n, 4, r, err) != 0) return -1;
    if (r.reason) return refuse();
    const auto t1 = P.t_h2d;
    size_t& bytes = P.bytes;
    const char* d_text = P.text;
    const int64_t N = P.N;
    unsigned long long* d_err = P.err;
    const int64_t *ops = P.ops, *ch = P.ch, *it_pos = P.it_pos;
    const int64_t n_ops = P.n_ops, n_ch = P.n_ch, n_it = P.n_it;
    int64_t *deep, n_deep = 0;
    JTB_OK(P.select(P.forms, P.nf, EdnAtDepth{d_text, P.depth, P.base + 3}, &deep, &n_deep));
    const int64_t n_m = n_it + n_deep;   // candidate members
    if (n_m >= INT_MAX - 2) {
        r.reason = "more than 2^31 - 3 set members";
        return refuse();
    }

    // ---- 5, 6: ops, :value elements, keys, members ------------------------------------------------------------------
    SetOp* op;
    int32_t *mop, *mval;
    JTB_OK(A.alloc(&op, (size_t)n_ops));
    JTB_OK(A.alloc(&mop, (size_t)n_m));
    JTB_OK(A.alloc(&mval, (size_t)n_m));
    if (n_ops) {
        set_op_kernel<<<edn_blocks(n_ops), T, 0, st>>>(d_text, N, ops, n_ops, ch, P.n_child, P.field, op, d_err);
        if (n_it) set_item_kernel<<<edn_blocks(n_it), T, 0, st>>>(ops, n_ops, ch, n_ch, it_pos, n_it, op);
        set_event_kernel<<<edn_blocks(n_ops), T, 0, st>>>(d_text, N, n_ops, ch, it_pos, op, d_err);
        if (n_m)
            set_member_kernel<<<edn_blocks(n_m), T, 0, st>>>(d_text, N, ops, n_ops, it_pos, n_it, deep, n_deep, op,
                                                             mop, mval, d_err);
        JTB_OK(cudaGetLastError());
    }
    JTB_OK(P.error_word(&w));
    if (refused_word()) return refuse();

    // ---- 7: events, the key partition, payload offsets ----------------------------------------------------------------
    int32_t *keyed, *unkeyed, *sop, *spos, *order = nullptr;
    int64_t n_keyed = 0, n_unkeyed = 0, *d_key, *d_off, *d_ids;
    JTB_OK(A.alloc(&keyed, (size_t)n_ops));
    JTB_OK(A.alloc(&unkeyed, (size_t)n_ops));
    auto oi = thrust::counting_iterator<int32_t>(0);
    JTB_OK(P.count(oi, n_ops, SetKept{op, 1}, &n_keyed));
    JTB_OK(P.select_into(oi, n_ops, SetKept{op, 1}, keyed));
    JTB_OK(P.count(oi, n_ops, SetKept{op, 0}, &n_unkeyed));
    JTB_OK(P.select_into(oi, n_ops, SetKept{op, 0}, unkeyed));
    const int64_t n_events = n_keyed + n_unkeyed;
    JTB_OK(A.alloc(&d_key, (size_t)n_keyed));
    JTB_OK(A.alloc(&d_off, (size_t)n_keyed + 1));
    JTB_OK(A.alloc(&d_ids, (size_t)n_keyed + 1));
    JTB_OK(A.alloc(&sop, (size_t)n_events));
    JTB_OK(A.alloc(&spos, (size_t)n_ops));
    int32_t runs = 0;
    if (n_keyed) {
        set_key_kernel<<<edn_blocks(n_keyed), T, 0, st>>>(op, keyed, n_keyed, d_key);
        JTB_OK(cudaGetLastError());
        if (partition_by_key_device(st, A, n_keyed, d_key, &order, d_off, d_ids, (int32_t)n_keyed, &runs, err) != 0)
            return -1;
    }
    int64_t *poff_incl, n_payload = 0;
    JTB_OK(A.alloc(&poff_incl, (size_t)n_events));
    EdnEvents e;
    JTB_OK(A.alloc(&e.type, (size_t)n_events));
    JTB_OK(A.alloc(&e.f, (size_t)n_events));
    JTB_OK(A.alloc(&e.flags, (size_t)n_events));
    JTB_OK(A.alloc(&e.process, (size_t)n_events));
    JTB_OK(A.alloc(&e.index, (size_t)n_events));
    JTB_OK(A.alloc(&e.a, (size_t)n_events));
    JTB_OK(A.alloc(&e.b, (size_t)n_events));
    JTB_OK(A.alloc(&e.c, (size_t)n_events));
    JTB_OK(A.alloc(&e.payload_len, (size_t)n_events));
    JTB_OK(A.alloc(&e.time_ns, (size_t)n_events));
    JTB_OK(A.alloc(&e.payload_off, (size_t)n_events));
    if (n_events) {
        set_order_kernel<<<edn_blocks(n_events), T, 0, st>>>(keyed, order, n_keyed, unkeyed, n_events, sop, spos);
        JTB_OK(cudaGetLastError());
        auto plen = thrust::make_transform_iterator(thrust::counting_iterator<int64_t>(0), SetPlen{op, sop});
        JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, bytes, plen, poff_incl, n_events, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceScan::InclusiveSum(P.tmp, bytes, plen, poff_incl, n_events, st));
        set_write_events_kernel<<<edn_blocks(n_events), T, 0, st>>>(op, sop, n_events, poff_incl, e);
        JTB_OK(cudaGetLastError());
        JTB_OK(P.fetch(&n_payload, poff_incl + n_events - 1));
    }

    // ---- 8: the payload: members sorted by (event, member) for sets, by event for vectors and lists ---------------
    uint64_t *k0, *k1;
    int32_t* v1;
    JTB_OK(A.alloc(&k0, (size_t)n_m));
    JTB_OK(A.alloc(&k1, (size_t)n_m));
    JTB_OK(A.alloc(&v1, (size_t)n_m));
    if (n_payload) {
        int ev_bits = 0;   // 2^ev_bits > n_events: a member's key stays below a non-member's
        while (ev_bits < 32 && (1ll << ev_bits) <= n_events) ++ev_bits;
        set_sort_key_kernel<<<edn_blocks(n_m), T, 0, st>>>(mop, mval, n_m, op, spos, k0);
        JTB_OK(cudaGetLastError());
        JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, k0, k1, mval, v1, n_m, 0, 32 + ev_bits, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceRadixSort::SortPairs(P.tmp, bytes, k0, k1, mval, v1, n_m, 0, 32 + ev_bits, st));
        set_repeat_kernel<<<edn_blocks(n_payload), T, 0, st>>>(k1, n_payload, op, sop, ops, d_err);
        JTB_OK(cudaGetLastError());
        JTB_OK(P.error_word(&w));
        if (refused_word()) return refuse();
    }
    JTB_OK(cudaEventRecord(ev1, st));
    JTB_OK(cudaStreamSynchronize(st));
    const auto t2 = Clock::now();
    float ms = 0;
    JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));

    // ---- the arrays, copied into page-locked host memory the library owns ---------------------------------------------
    const int32_t n_shards = n_events == 0 ? 1 : runs + (n_unkeyed ? 1 : 0);
    jtb_history& h = out->history;
    bool ok = true;
    auto host = [&](void** p, size_t bytes_) {
        *p = jtb_host_alloc(bytes_);
        ok = ok && *p;
    };
    host((void**)&h.type, n_events);
    host((void**)&h.f, n_events);
    host((void**)&h.flags, n_events);
    host((void**)&h.process, n_events * 4);
    host((void**)&h.index, n_events * 4);
    host((void**)&h.time_ns, n_events * 8);
    host((void**)&h.a, n_events * 4);
    host((void**)&h.b, n_events * 4);
    host((void**)&h.c, n_events * 4);
    host((void**)&h.payload_off, n_events * 8);
    host((void**)&h.payload_len, n_events * 4);
    host((void**)&h.payload, n_payload * 4);
    host((void**)&h.shard_off, ((size_t)n_shards + 1) * 8);
    host((void**)&h.key_ids, (size_t)n_shards * 8);
    if (!ok) {
        jtb_edn_history_release(out);
        return input_error(err, "jtb_host_alloc failed for the flattened history");
    }
    auto d2h = [&](void* dst, const void* src, size_t bytes_) -> cudaError_t {
        return bytes_ ? cudaMemcpyAsync(dst, src, bytes_, cudaMemcpyDeviceToHost, st) : cudaSuccess;
    };
    cudaError_t ce = cudaSuccess;
    const size_t ne = (size_t)n_events;
    for (auto [dst, src, nbytes] : {std::tuple<void*, const void*, size_t>{(void*)h.type, e.type, ne},
                                    {(void*)h.f, e.f, ne}, {(void*)h.flags, e.flags, ne},
                                    {(void*)h.process, e.process, ne * 4}, {(void*)h.index, e.index, ne * 4},
                                    {(void*)h.time_ns, e.time_ns, ne * 8}, {(void*)h.a, e.a, ne * 4},
                                    {(void*)h.b, e.b, ne * 4}, {(void*)h.c, e.c, ne * 4},
                                    {(void*)h.payload_off, e.payload_off, ne * 8},
                                    {(void*)h.payload_len, e.payload_len, ne * 4},
                                    {(void*)h.payload, v1, (size_t)n_payload * 4},
                                    {(void*)h.shard_off, d_off, (size_t)runs * 8},
                                    {(void*)h.key_ids, d_ids, (size_t)runs * 8}})
        if (ce == cudaSuccess) ce = d2h(dst, src, nbytes);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) {
        jtb_edn_history_release(out);
        err = std::string("copying the history back: ") + cudaGetErrorString(ce);
        return -1;
    }
    int64_t* so = (int64_t*)h.shard_off;
    int64_t* ki = (int64_t*)h.key_ids;
    if (runs < n_shards) {   // the unkeyed events (or an empty history): the last shard, key id -1
        so[runs] = n_keyed;
        ki[runs] = -1;
    }
    so[n_shards] = n_events;
    h.n_events = n_events;
    h.n_payload = n_payload;
    h.n_shards = n_shards;
    out->n_ops = n_ops;
    const auto t3 = Clock::now();
    out->seconds_h2d = std::chrono::duration<double>(t1 - t0).count();
    out->seconds_kernel = ms * 1e-3;
    out->seconds_d2h = std::chrono::duration<double>(t3 - t2).count();
    out->seconds_total = std::chrono::duration<double>(t3 - t0).count();
    return 0;
}

}  // namespace jtb
