// jtb_edn.cuh — K18: a stored ledger history.edn read on the device into the flattened ledger forms.
//
// Semantics (include/jtb_check.h, DESIGN.md "K18 stored-history reader"): the arrays are exactly those of
// `edn.read_history(text)` followed by `history.flatten_ops(ops, form)` for the "bank", "ledger-counters" and
// "ledger-lookups" forms; where that Python path raises, the call returns rc < 0.  The EDN read is Jepsen's store
// subset: one op map per top-level form (optionally tagged) or one top-level vector of them; `;` comments, `#_` discard,
// character literals and floats where an integer is read are refused as unsupported.
//
// Passes, each over the whole buffer with no thread or warp per op line:
//   1. string state: a quote is unescaped when an even run of backslashes precedes it; a XOR scan of those quotes
//      gives, per byte, whether it lies inside a string.
//   2. depth: an inclusive sum of +1 per open ([ { ( and the { of #{) and -1 per close outside strings.  Bracket
//      pairing is checked by a stable radix sort of the brackets by level: each level then alternates open, close.
//   3. form starts (opens, strings, tokens that are not tags) at depth <= 3 (K20, jtb_set_edn.cuh, reads one level
//      deeper) are compacted; the top-level count decides
//      between one-op-per-form and one-vector files (base depth 0 or 1).  Ops are the form starts at the base depth,
//      their keys and values those at base + 1, micro-ops those at base + 2.
//   4. one thread per map entry records where each of the seven op keys' value is; a thread per op then reads those
//      few scalars (O(1) work, whatever the length of the line).
//   5. one thread per micro-op parses its [tag id {...}]; the pending tag of an empty :ok lookup comes from the previous
//      op of its process (a stable radix sort of the client ops by process); payload offsets come from cub scans and a
//      last pass writes the events and the payload in place.
#pragma once
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdint>
#include <cstring>
#include <string>
#include <tuple>

#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "../../include/jtb_check.h"
#include "jtb_call.cuh"

namespace jtb {

// error codes: the device keeps the smallest (byte position << 8 | code), so the first error in the file is reported
enum EdnErr : uint32_t {
    EE_STRING = 1, EE_COMMENT, EE_CHAR, EE_DISCARD, EE_BRACKETS, EE_NOT_MAP, EE_ODD_MAP, EE_TYPE, EE_F, EE_NUMBER,
    EE_INDEX, EE_TIME, EE_PROCESS, EE_FINAL, EE_VALUE, EE_EMPTY_TXN, EE_TAG, EE_MICRO_OP, EE_ACCOUNT, EE_NO_ID,
    EE_INT64, EE_INT32, EE_FIELD, EE_COUNT
};
inline const char* edn_err_text(uint32_t c) {
    static const char* m[EE_COUNT] = {
        "", "unterminated string", "unsupported EDN: ';' comment", "unsupported EDN: character literal",
        "unsupported EDN: #_ discard", "unbalanced or mismatched brackets", "history entries must be maps",
        "map with odd number of forms", "unknown or missing :type", ":f other than :txn",
        "unsupported EDN: a number that is not an integer", ":index is not an int32", ":time is not an int64",
        ":process does not fit in int32", "unsupported :final? value", ":value of a txn is not a vector or nil",
        "a txn without micro-ops", "unknown txn micro-op", "a micro-op that is not [tag id value]",
        "account outside [0, 2^30) or not an integer", "a transfer without an id", "an id or counter outside int64",
        "a value does not fit its int32 column", "a transfer map field that is missing or not an integer"};
    return c < EE_COUNT ? m[c] : "unknown error";
}

enum : uint8_t { SK_NIL = 1, SK_TRUE, SK_FALSE, SK_INT, SK_BIG, SK_KW, SK_BADNUM, SK_OTHER };   // 0: absent
enum : uint8_t { TG_NONE = 0, TG_R, TG_T, TG_LT, TG_OTHER, TG_PENDING };
enum : uint8_t { PM_NONE = 0, PM_BANK, PM_TRIPLES, PM_RECORDS };
// an op's :value as flatten_ops sees it: nil or absent, false or 0 (falsy, not iterable), an empty collection or "",
// a non-empty vector or list
enum : uint8_t { VK_NIL = 0, VK_FALSY, VK_EMPTY, VK_VEC };
enum { EK_TYPE = 0, EK_F, EK_PROCESS, EK_INDEX, EK_TIME, EK_FINAL, EK_VALUE, EK_N };
enum { MV_DEBIT = 0, MV_CREDIT, MV_AMOUNT, MV_DEBITS, MV_CREDITS, MV_N };

struct EdnOp {
    int64_t time;
    int64_t plen;          // payload entries (sum over the micro-ops); -1 none
    int32_t process, index;
    int32_t value_child;   // the child (entry) index of the :value form, -1 nil or absent
    int32_t first_item, n_items;
    int32_t a, b, c;
    uint8_t type, flags, client, tag, keep, f, pm, vkind;
};

struct EdnItem {
    int64_t id;
    int64_t v[MV_N];
    int32_t op;            // -1: not a micro-op of a client op's :value
    uint8_t vector, n_elems, tag, id_kind, map_kind, vk[MV_N];
};

__device__ __forceinline__ bool edn_ws(char c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n' || c == ','; }
__device__ __forceinline__ bool edn_open(char c) { return c == '[' || c == '{' || c == '('; }
__device__ __forceinline__ bool edn_close(char c) { return c == ']' || c == '}' || c == ')'; }
__device__ __forceinline__ bool edn_delim(char c) {
    return edn_ws(c) || edn_open(c) || edn_close(c) || c == '"' || c == ';';
}

__device__ __forceinline__ void edn_fail(unsigned long long* err, int64_t pos, uint32_t code) {
    atomicMin(err, ((unsigned long long)pos << 8) | code);
}

// the token at p is exactly the literal s (length n)
__device__ __forceinline__ bool edn_is(const char* t, int64_t p, const char* s, int n) {
    for (int k = 0; k < n; ++k)
        if (t[p + k] != s[k]) return false;
    return edn_delim(t[p + n]);
}

__device__ __forceinline__ int64_t edn_token_end(const char* t, int64_t p, int64_t n) {
    while (p < n && !edn_delim(t[p])) ++p;
    return p;
}
__device__ __forceinline__ int64_t edn_skip_ws(const char* t, int64_t p, int64_t n) {
    while (p < n && edn_ws(t[p])) ++p;
    return p;
}

// the position after the form at p (tags included: a tag and its value are one form)
__device__ int64_t edn_skip_form(const char* t, int64_t p, int64_t n) {
    while (p < n && t[p] == '#' && t[p + 1] != '{') p = edn_skip_ws(t, edn_token_end(t, p + 1, n), n);
    if (p >= n) return n;
    if (t[p] == '#') ++p;
    const char c = t[p];
    if (c == '"') {
        for (++p; p < n && t[p] != '"'; ++p)
            if (t[p] == '\\') ++p;
        return p + 1;
    }
    if (!edn_open(c)) return edn_token_end(t, p, n);
    int d = 0;
    for (; p < n; ++p) {
        const char x = t[p];
        if (x == '"') {
            for (++p; p < n && t[p] != '"'; ++p)
                if (t[p] == '\\') ++p;
        } else if (edn_open(x)) {
            ++d;
        } else if (edn_close(x) && --d == 0) {
            return p + 1;
        }
    }
    return n;
}

// the form a tagged literal at p tags (edn.py drops the tag); p itself when it is not one
__device__ __forceinline__ int64_t edn_untag(const char* t, int64_t p, int64_t n) {
    while (p < n && t[p] == '#' && t[p + 1] != '{' && t[p + 1] != '_') p = edn_skip_ws(t, edn_token_end(t, p + 1, n), n);
    return p;
}

// a scalar at p: SK_* and, for SK_INT, its value
__device__ uint8_t edn_scalar(const char* t, int64_t p, int64_t n, int64_t* v) {
    p = edn_untag(t, p, n);
    if (p >= n) return SK_OTHER;
    const char c = t[p];
    if (edn_open(c) || c == '"' || c == '#') return SK_OTHER;
    const int64_t e = edn_token_end(t, p, n);
    if (c == ':') return SK_KW;
    if (edn_is(t, p, "nil", 3)) return SK_NIL;
    if (edn_is(t, p, "true", 4)) return SK_TRUE;
    if (edn_is(t, p, "false", 5)) return SK_FALSE;
    int64_t q = p;
    const bool neg = c == '-';
    if (c == '+' || c == '-') ++q;
    if (q >= e || t[q] < '0' || t[q] > '9') return SK_OTHER;   // a symbol
    unsigned long long m = 0;
    bool big = false;
    for (; q < e; ++q) {
        const char d = t[q];
        if (d == 'N' && q == e - 1) break;
        if (d < '0' || d > '9') return SK_BADNUM;
        if (!big) {
            if (m > (~0ull - 9) / 10) big = true;
            else m = m * 10 + (unsigned long long)(d - '0');
        }
    }
    if (big || m > (neg ? (1ull << 63) : (1ull << 63) - 1)) return SK_BIG;
    *v = neg ? (int64_t)(0ull - m) : (int64_t)m;
    return SK_INT;
}

// Python truthiness of the form at p (nil, false, 0, "" and empty collections are false); -1: a number edn.py reads
// as a float, which the reader does not
__device__ int edn_truthy(const char* t, int64_t p, int64_t n) {
    p = edn_untag(t, p, n);
    if (p >= n) return 0;
    if (t[p] == '"') return t[p + 1] != '"';
    const int64_t q = t[p] == '#' ? p + 1 : p;   // #{ a set
    if (edn_open(t[q])) {
        const int64_t r = edn_skip_ws(t, q + 1, n);
        return r < n && !edn_close(t[r]);
    }
    int64_t v = 0;
    const uint8_t k = edn_scalar(t, p, n, &v);
    if (k == SK_BADNUM) return -1;
    if (k == SK_NIL || k == SK_FALSE) return 0;
    return k == SK_INT ? v != 0 : 1;
}

// ---- pass 1 and 2: string state and depth ---------------------------------------------------------------------------
struct EdnQuote {   // 1 at an unescaped quote
    const char* t;
    __device__ uint8_t operator()(int64_t i) const {
        if (t[i] != '"') return 0;
        int64_t j = i - 1;
        while (j >= 0 && t[j] == '\\') --j;
        return ((i - 1 - j) & 1) ? 0 : 1;
    }
};
struct EdnXor {
    __device__ uint8_t operator()(uint8_t a, uint8_t b) const { return a ^ b; }
};
struct EdnDelta {   // +1 open, -1 close, outside strings (par: inclusive quote parity; a closing quote has parity 0)
    const char* t;
    const uint8_t* par;
    __device__ int operator()(int64_t i) const {
        const char c = t[i];
        if (par[i] || c == '"') return 0;
        return edn_open(c) ? 1 : edn_close(c) ? -1 : 0;
    }
};

__device__ __forceinline__ bool edn_outside(const char* t, const uint8_t* par, int64_t i) {
    return !par[i] && t[i] != '"';
}

__global__ void edn_byte_check_kernel(const char* t, const uint8_t* par, const int* depth, int64_t n,
                                      unsigned long long* err) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        if (!edn_outside(t, par, i)) continue;
        const char c = t[i];
        if (c == ';') edn_fail(err, i, EE_COMMENT);
        else if (c == '\\') edn_fail(err, i, EE_CHAR);
        else if (c == '#' && t[i + 1] == '_') edn_fail(err, i, EE_DISCARD);
        else if (edn_close(c) && depth[i] < 0) edn_fail(err, i, EE_BRACKETS);
    }
}

struct EdnIsBracket {
    const char* t;
    const uint8_t* par;
    __device__ bool operator()(int64_t i) const {
        return edn_outside(t, par, i) && (edn_open(t[i]) || edn_close(t[i]));
    }
};

__global__ void edn_bracket_level_kernel(const char* t, const int* depth, const int64_t* br, int64_t nb,
                                         uint32_t* level) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= nb) return;
    const int64_t i = br[k];
    const int d = edn_open(t[i]) ? depth[i] : depth[i] + 1;
    level[k] = (uint32_t)max(d, 0);
}

// sorted by (level, position): pairs (2k, 2k+1) are an open and the close that matches it
__global__ void edn_bracket_pair_kernel(const char* t, const uint32_t* level, const int64_t* pos, int64_t nb,
                                        unsigned long long* err) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (2 * k >= nb) return;
    const int64_t i = pos[2 * k];
    if (2 * k + 1 >= nb) { edn_fail(err, i, EE_BRACKETS); return; }
    const int64_t j = pos[2 * k + 1];
    const char o = t[i], c = t[j];
    const bool ok = level[2 * k] == level[2 * k + 1] && edn_open(o) &&
                    ((o == '[' && c == ']') || (o == '{' && c == '}') || (o == '(' && c == ')'));
    if (!ok) edn_fail(err, min(i, j), EE_BRACKETS);
}

// ---- pass 3: form starts --------------------------------------------------------------------------------------------
__device__ __forceinline__ int edn_depth_before(const char* t, const int* depth, int64_t i) {
    return depth[i] - (edn_open(t[i]) ? 1 : 0);
}

struct EdnFormStart {   // an open, an opening quote or a token that is not a tag, at depth <= max_depth
    const char* t;
    const uint8_t* par;
    const int* depth;
    int max_depth;      // 3 for the ledger forms; the set form's members sit one level deeper
    __device__ bool operator()(int64_t i) const {
        const char c = t[i];
        if (par[i]) return c == '"' && (i == 0 || !par[i - 1]) && depth[i] <= max_depth;
        if (c == '"') return false;
        if (edn_open(c)) return depth[i] - 1 <= max_depth;
        if (edn_delim(c) || c == '#') return false;
        if (i > 0 && !edn_delim(t[i - 1])) return false;
        return depth[i] <= max_depth;
    }
};

struct EdnAtDepth {
    const char* t;
    const int* depth;
    int d;
    __device__ bool operator()(int64_t i) const { return edn_depth_before(t, depth, i) == d; }
};

__global__ void edn_top_kernel(const char* t, const int* depth, const int64_t* forms, int64_t nf, int* n_top) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int top = k < nf && edn_depth_before(t, depth, forms[k]) == 0;
    const int cnt = __syncthreads_count(top);
    if (threadIdx.x == 0 && cnt) atomicAdd(n_top, cnt);
}

// index of the last element of sorted a[0, n) that is <= x, -1 none
__device__ __forceinline__ int64_t edn_floor(const int64_t* a, int64_t n, int64_t x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] <= x) lo = mid + 1;
        else hi = mid;
    }
    return lo - 1;
}

// ---- pass 4: op keys and fields -------------------------------------------------------------------------------------
__global__ void edn_child_kernel(const int64_t* ops, int64_t n_ops, const int64_t* ch, int64_t n_ch, int32_t* ch_op,
                                 int32_t* first_child, int32_t* n_child) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n_ch) return;
    const int32_t o = (int32_t)edn_floor(ops, n_ops, ch[j]);
    ch_op[j] = o;
    if (o < 0) return;
    atomicMin(&first_child[o], (int32_t)j);
    atomicAdd(&n_child[o], 1);
}

__global__ void edn_key_kernel(const char* t, const int64_t* ch, int64_t n_ch, const int32_t* ch_op,
                               const int32_t* first_child, int32_t* field) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= n_ch) return;
    const int32_t o = ch_op[j];
    if (o < 0 || ((j - first_child[o]) & 1)) return;   // a value
    if (j + 1 >= n_ch || ch_op[j + 1] != o) return;     // the last form of an odd map: a key without a value
    const int64_t p = ch[j];
    if (t[p] != ':') return;
    int k = -1;
    if (edn_is(t, p, ":type", 5)) k = EK_TYPE;
    else if (edn_is(t, p, ":f", 2)) k = EK_F;
    else if (edn_is(t, p, ":process", 8)) k = EK_PROCESS;
    else if (edn_is(t, p, ":index", 6)) k = EK_INDEX;
    else if (edn_is(t, p, ":time", 5)) k = EK_TIME;
    else if (edn_is(t, p, ":final?", 7)) k = EK_FINAL;
    else if (edn_is(t, p, ":value", 6)) k = EK_VALUE;
    if (k >= 0) atomicMax(&field[(int64_t)o * EK_N + k], (int32_t)j + 2);   // the value's index + 1; the last key wins
}

// The fields every form reads from op o's map: :type, :time, :process and, for a client op, :index and :final?.  False
// when the map has an odd number of forms (refused; the op stays a non-client op, so no later pass reads its fields).
__device__ __forceinline__ bool edn_op_fields(const char* t, int64_t n, int64_t o, int64_t pos, const int64_t* ch,
                                              const int32_t* n_child, const int32_t* fo, EdnOp& op,
                                              unsigned long long* err) {
    int64_t v = 0;
    if (t[pos] != '{' || (pos > 0 && t[pos - 1] == '#')) edn_fail(err, pos, EE_NOT_MAP);
    if (n_child[o] & 1) {
        edn_fail(err, pos, EE_ODD_MAP);
        return false;
    }
    // :type (every op)
    if (!fo[EK_TYPE]) {
        edn_fail(err, pos, EE_TYPE);
    } else {
        const int64_t p = ch[fo[EK_TYPE] - 1];
        if (edn_is(t, p, ":invoke", 7)) op.type = JTB_T_INVOKE;
        else if (edn_is(t, p, ":ok", 3)) op.type = JTB_T_OK;
        else if (edn_is(t, p, ":fail", 5)) op.type = JTB_T_FAIL;
        else if (edn_is(t, p, ":info", 5)) op.type = JTB_T_INFO;
        else edn_fail(err, p, EE_TYPE);
    }
    // :time (every op: int() of it), default: the op's position
    uint8_t time_kind = SK_INT;
    op.time = o;
    if (fo[EK_TIME]) {
        const int64_t p = ch[fo[EK_TIME] - 1];
        time_kind = edn_scalar(t, p, n, &v);
        if (time_kind == SK_INT) op.time = v;
        else if (time_kind == SK_BADNUM) edn_fail(err, p, EE_NUMBER);
        else if (time_kind != SK_BIG) edn_fail(err, p, EE_TIME);
    }
    // :process: an integer makes a client op; anything else is skipped
    if (fo[EK_PROCESS]) {
        const int64_t p = ch[fo[EK_PROCESS] - 1];
        const uint8_t k = edn_scalar(t, p, n, &v);
        if (k == SK_BADNUM) edn_fail(err, p, EE_NUMBER);
        if (k == SK_BIG || (k == SK_INT && (v < INT_MIN || v > INT_MAX))) edn_fail(err, p, EE_PROCESS);
        if (k == SK_INT) { op.client = 1; op.process = (int32_t)v; }
    }
    if (op.client) {
        if (time_kind == SK_BIG) edn_fail(err, ch[fo[EK_TIME] - 1], EE_TIME);
        op.index = (int32_t)o;
        if (fo[EK_INDEX]) {
            const int64_t p = ch[fo[EK_INDEX] - 1];
            const uint8_t k = edn_scalar(t, p, n, &v);
            if (k == SK_BADNUM) edn_fail(err, p, EE_NUMBER);
            else if (k != SK_INT || v < INT_MIN || v > INT_MAX) edn_fail(err, p, EE_INDEX);
            else op.index = (int32_t)v;
        }
        if (fo[EK_FINAL]) {   // truthiness, as flatten_ops tests it
            const int64_t p = ch[fo[EK_FINAL] - 1];
            const int truthy = edn_truthy(t, p, n);
            if (truthy < 0) edn_fail(err, p, EE_NUMBER);
            else if (truthy) op.flags = JTB_FLAG_FINAL;
        }
    }
    return true;
}

__global__ void edn_op_kernel(const char* t, int64_t n, const int64_t* ops, int64_t n_ops, const int64_t* ch,
                              const int32_t* n_child, const int32_t* field, EdnOp* out, unsigned long long* err) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= n_ops) return;
    const int64_t pos = ops[o];
    EdnOp op{};
    op.value_child = -1;
    op.first_item = INT_MAX;
    op.plen = -1;
    const int32_t* fo = field + o * EK_N;
    int64_t v = 0;
    if (!edn_op_fields(t, n, o, pos, ch, n_child, fo, op, err)) {
        out[o] = op;
        return;
    }
    if (op.client) {
        if (!fo[EK_F] || !edn_is(t, ch[fo[EK_F] - 1], ":txn", 4)) edn_fail(err, fo[EK_F] ? ch[fo[EK_F] - 1] : pos, EE_F);
        op.vkind = VK_NIL;
        if (fo[EK_VALUE]) {
            const int64_t p = ch[fo[EK_VALUE] - 1];
            const int truthy = edn_truthy(t, p, n);
            if ((t[p] == '[' || t[p] == '(') && !(t[p - 1] == '#')) {
                op.value_child = fo[EK_VALUE] - 1;
                op.vkind = truthy ? VK_VEC : VK_EMPTY;
            } else if (truthy == 0) {   // nil, false, 0, "", an empty map or set
                const uint8_t k = edn_scalar(t, p, n, &v);
                op.vkind = k == SK_NIL ? VK_NIL : (k == SK_FALSE || k == SK_INT) ? VK_FALSY : VK_EMPTY;
            } else {
                edn_fail(err, p, EE_VALUE);   // a non-empty map, set, string or scalar: refused
            }
        }
    }
    out[o] = op;
}

// ---- pass 5: micro-ops ----------------------------------------------------------------------------------------------
__device__ void edn_parse_map(const char* t, int64_t p, int64_t n, EdnItem& it, int64_t pos,
                              unsigned long long* err) {
    int64_t q = p + 1;
    for (;;) {
        q = edn_skip_ws(t, q, n);
        if (q >= n || t[q] == '}') return;
        int k = -1;
        if (t[q] == ':') {
            if (edn_is(t, q, ":debit-acct", 11)) k = MV_DEBIT;
            else if (edn_is(t, q, ":credit-acct", 12)) k = MV_CREDIT;
            else if (edn_is(t, q, ":amount", 7)) k = MV_AMOUNT;
            else if (edn_is(t, q, ":debits-posted", 14)) k = MV_DEBITS;
            else if (edn_is(t, q, ":credits-posted", 15)) k = MV_CREDITS;
        }
        q = edn_skip_ws(t, edn_skip_form(t, q, n), n);
        if (q >= n || t[q] == '}') { edn_fail(err, pos, EE_ODD_MAP); return; }
        if (k >= 0) it.vk[k] = edn_scalar(t, q, n, &it.v[k]);   // a tagged value is read through its tag
        q = edn_skip_form(t, q, n);
    }
}

__global__ void edn_item_kernel(const char* t, int64_t n, const int64_t* ops, int64_t n_ops, const int64_t* ch,
                                int64_t n_ch, const int64_t* items, int64_t n_items, EdnOp* op, EdnItem* out,
                                unsigned long long* err) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_items) return;
    const int64_t pos = items[k];
    EdnItem it{};
    it.op = -1;
    const int64_t o = edn_floor(ops, n_ops, pos);
    if (o < 0 || !op[o].client || op[o].value_child < 0 || edn_floor(ch, n_ch, pos) != op[o].value_child) {
        out[k] = it;
        return;
    }
    it.op = (int32_t)o;
    atomicMin(&op[o].first_item, (int32_t)k);
    atomicAdd(&op[o].n_items, 1);
    const char c = t[pos];
    if ((c == '[' || c == '(') && !(t[pos - 1] == '#')) {
        it.vector = 1;
        int64_t q = pos + 1;
        int ne = 0;
        for (;;) {
            q = edn_untag(t, edn_skip_ws(t, q, n), n);
            if (q >= n || edn_close(t[q])) break;
            if (ne == 0) {
                it.tag = edn_is(t, q, ":r", 2) ? TG_R : edn_is(t, q, ":t", 2) ? TG_T
                         : edn_is(t, q, ":l-t", 4) ? TG_LT : TG_OTHER;
            } else if (ne == 1) {
                it.id_kind = edn_scalar(t, q, n, &it.id);
            } else if (ne == 2) {
                if (t[q] == '{' && t[q - 1] != '#') {
                    it.map_kind = 1;
                    edn_parse_map(t, q, n, it, pos, err);
                } else {
                    int64_t dummy;
                    it.map_kind = edn_scalar(t, q, n, &dummy) == SK_NIL ? 0 : 2;
                }
            }
            q = edn_skip_form(t, q, n);
            ne = min(ne + 1, 255);
        }
        it.n_elems = (uint8_t)ne;
    }
    out[k] = it;
}

// the op's tag from its first micro-op; an empty value: pending (ledger-lookups, not an invoke) or an error
__global__ void edn_tag_kernel(const int64_t* ops, int64_t n_ops, EdnOp* op, const EdnItem* items, const int64_t* it_pos,
                               int form, unsigned long long* err) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= n_ops || !op[o].client) return;
    if (op[o].n_items > 0) {
        const EdnItem& f = items[op[o].first_item];
        const int64_t p = it_pos[op[o].first_item];
        if (!f.vector || f.n_elems == 0) edn_fail(err, p, EE_MICRO_OP);
        else if (f.tag == TG_OTHER) edn_fail(err, p, EE_TAG);
        op[o].tag = f.tag;
    } else if (form == JTB_FORM_LEDGER_LOOKUPS && op[o].type != JTB_T_INVOKE) {
        op[o].tag = TG_PENDING;
    } else {
        edn_fail(err, ops[o], EE_EMPTY_TXN);
    }
}

struct EdnIsClient {
    const EdnOp* op;
    __device__ bool operator()(int32_t o) const { return op[o].client != 0; }
};

__global__ void edn_proc_key_kernel(const EdnOp* op, const int32_t* cl, int64_t n, int32_t* key) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s < n) key[s] = op[cl[s]].process;
}

// sorted by (process, position): an empty :ok lookup takes the tag of its process's previous op when that is an invoke
__global__ void edn_pending_kernel(const int64_t* ops, EdnOp* op, const int32_t* key, const int32_t* sorted, int64_t n,
                                   unsigned long long* err) {
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int32_t o = sorted[s];
    if (op[o].tag != TG_PENDING) return;
    const int32_t prev = s > 0 && key[s - 1] == key[s] ? sorted[s - 1] : -1;
    if (prev < 0 || op[prev].type != JTB_T_INVOKE) { edn_fail(err, ops[o], EE_EMPTY_TXN); return; }
    const uint8_t tag = op[prev].tag;
    // flatten_ops unpacks value[0] of a transfer and iterates the value of an :ok read: both raise on an empty value
    // (an :ok read of [] or {} is an empty read); the op keeps TG_PENDING, so no later pass reads its micro-ops
    if (tag == TG_T || (tag == TG_R && op[o].type == JTB_T_OK && op[o].vkind != VK_EMPTY)) {
        edn_fail(err, ops[o], EE_EMPTY_TXN);
        return;
    }
    op[o].tag = tag;
}

__device__ __forceinline__ bool edn_i32(uint8_t k, int64_t v) { return k == SK_INT && v >= INT_MIN && v <= INT_MAX; }

// which events the ops become, their payload mode and a, b, c (the first micro-op of a transfer)
__global__ void edn_event_kernel(const int64_t* ops, int64_t n_ops, EdnOp* op, const EdnItem* items,
                                 const int64_t* it_pos, int form, unsigned long long* err,
                                 unsigned long long* multi) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= n_ops) return;
    EdnOp& x = op[o];
    x.keep = 0;
    if (!x.client || x.tag == TG_PENDING || x.tag == TG_NONE || x.tag == TG_OTHER) return;   // errors reported
    if (x.tag == TG_LT && form != JTB_FORM_LEDGER_LOOKUPS) return;   // dropped, as ledger->bank drops it
    x.keep = 1;
    x.f = x.tag == TG_R ? JTB_F_READ : x.tag == TG_T ? JTB_F_TRANSFER : JTB_F_LOOKUP;
    x.pm = PM_NONE;
    if (x.tag == TG_R && x.type == JTB_T_OK) x.pm = form == JTB_FORM_BANK ? PM_BANK : PM_TRIPLES;
    if (form == JTB_FORM_LEDGER_LOOKUPS && ((x.tag == TG_T && x.type == JTB_T_INVOKE) || (x.tag == TG_LT && x.type == JTB_T_OK)))
        x.pm = PM_RECORDS;
    x.plen = x.pm == PM_NONE ? -1 : 0;
    if (x.tag == TG_T) {
        if (x.n_items == 0) { edn_fail(err, ops[o], EE_EMPTY_TXN); x.keep = 0; return; }
        const EdnItem& f = items[x.first_item];
        const int64_t p = it_pos[x.first_item];
        if (f.n_elems != 3) { edn_fail(err, p, EE_MICRO_OP); return; }
        if (f.map_kind != 1) { edn_fail(err, p, EE_FIELD); return; }
        const int mv[3] = {MV_AMOUNT, MV_DEBIT, MV_CREDIT};
        int32_t abc[3];
        for (int q = 0; q < 3; ++q) {
            const uint8_t k = f.vk[mv[q]];
            if (k == SK_INT || k == SK_BIG) {
                if (!edn_i32(k, f.v[mv[q]])) edn_fail(err, p, EE_INT32);
            } else {
                edn_fail(err, p, k == SK_BADNUM ? EE_NUMBER : EE_FIELD);
            }
            abc[q] = (int32_t)f.v[mv[q]];
        }
        x.a = abc[0]; x.b = abc[1]; x.c = abc[2];
        if (x.type == JTB_T_INVOKE && form != JTB_FORM_BANK && x.n_items > 1) atomicAdd(multi, 1ull);
    }
}

// each micro-op's payload entries (and its checks), summed into its op's payload length
__global__ void edn_contrib_kernel(const int64_t* it_pos, const EdnItem* items, int64_t n_items, EdnOp* op,
                                   int64_t* contrib, unsigned long long* err) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_items) return;
    const EdnItem& it = items[k];
    int64_t c = 0;
    const uint8_t pm = it.op >= 0 && op[it.op].keep ? op[it.op].pm : PM_NONE;
    const int64_t p = it_pos[k];
    if (pm != PM_NONE) {
        if (!it.vector || it.n_elems != 3) {
            edn_fail(err, p, EE_MICRO_OP);
        } else if (pm == PM_BANK) {
            if (it.id_kind == SK_BIG || (it.id_kind == SK_INT && !edn_i32(SK_INT, it.id))) edn_fail(err, p, EE_INT32);
            else if (it.id_kind != SK_INT) edn_fail(err, p, EE_ACCOUNT);
            if (it.map_kind == 2) edn_fail(err, p, EE_FIELD);
            // both counters present: credits - debits must fit int32; one of them absent or nil: the balance is NIL
            const bool both = it.map_kind == 1 && it.vk[MV_DEBITS] != 0 && it.vk[MV_DEBITS] != SK_NIL &&
                              it.vk[MV_CREDITS] != 0 && it.vk[MV_CREDITS] != SK_NIL;
            if (both) {
                for (int q = MV_DEBITS; q <= MV_CREDITS; ++q) {
                    const uint8_t vk = it.vk[q];
                    if (vk == SK_BIG) edn_fail(err, p, EE_INT64);
                    else if (vk == SK_BADNUM) edn_fail(err, p, EE_NUMBER);
                    else if (vk != SK_INT) edn_fail(err, p, EE_FIELD);
                }
                if (it.vk[MV_DEBITS] == SK_INT && it.vk[MV_CREDITS] == SK_INT) {
                    const __int128 d = (__int128)it.v[MV_CREDITS] - (__int128)it.v[MV_DEBITS];
                    if (d < INT_MIN || d > INT_MAX) edn_fail(err, p, EE_INT32);
                }
            }
            c = 2;
        } else if (pm == PM_TRIPLES) {
            if (it.id_kind != SK_INT || it.id < 0 || it.id >= (1ll << 30)) edn_fail(err, p, EE_ACCOUNT);
            if (it.map_kind == 2) edn_fail(err, p, EE_FIELD);
            if (it.map_kind == 1) {
                for (int q = MV_DEBITS; q <= MV_CREDITS; ++q) {
                    const uint8_t vk = it.vk[q];
                    if (vk == SK_INT) c += 3;
                    else if (vk == SK_BIG) edn_fail(err, p, EE_INT64);
                    else if (vk == SK_BADNUM) edn_fail(err, p, EE_NUMBER);
                    else if (vk != 0 && vk != SK_NIL) edn_fail(err, p, EE_FIELD);
                }
            }
        } else {   // PM_RECORDS
            if (it.map_kind == 2) edn_fail(err, p, EE_FIELD);
            if (it.map_kind == 1) {
                if (it.id_kind == 0 || it.id_kind == SK_NIL) edn_fail(err, p, EE_NO_ID);
                else if (it.id_kind == SK_BIG) edn_fail(err, p, EE_INT64);
                else if (it.id_kind != SK_INT) edn_fail(err, p, it.id_kind == SK_BADNUM ? EE_NUMBER : EE_FIELD);
                for (int q = MV_DEBIT; q <= MV_AMOUNT; ++q) {
                    const uint8_t vk = it.vk[q];
                    if (vk == SK_INT || vk == SK_BIG) {
                        if (!edn_i32(vk, it.v[q])) edn_fail(err, p, EE_INT32);
                    } else {
                        edn_fail(err, p, vk == SK_BADNUM ? EE_NUMBER : EE_FIELD);
                    }
                }
                c = 5;
            }
        }
        if (c) atomicAdd((unsigned long long*)&op[it.op].plen, (unsigned long long)c);
    }
    contrib[k] = c;
}

struct EdnKeep {
    const EdnOp* op;
    __device__ int64_t operator()(int64_t o) const { return op[o].keep; }
};
struct EdnPlen {
    const EdnOp* op;
    __device__ int64_t operator()(int64_t o) const { return op[o].keep && op[o].plen > 0 ? op[o].plen : 0; }
};

struct EdnEvents {
    uint8_t *type, *f, *flags;
    int32_t *process, *index, *a, *b, *c, *payload_len;
    int64_t *time_ns, *payload_off;
};

__global__ void edn_write_events_kernel(const EdnOp* op, int64_t n_ops, const int64_t* ev_incl,
                                        const int64_t* poff_incl, EdnEvents e) {
    const int64_t o = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (o >= n_ops || !op[o].keep) return;
    const EdnOp& x = op[o];
    const int64_t i = ev_incl[o] - 1;
    e.type[i] = x.type;
    e.f[i] = x.f;
    e.flags[i] = x.flags;
    e.process[i] = x.process;
    e.index[i] = x.index;
    e.time_ns[i] = x.time;
    e.a[i] = x.a;
    e.b[i] = x.b;
    e.c[i] = x.c;
    e.payload_off[i] = poff_incl[o] - (x.plen > 0 ? x.plen : 0);
    e.payload_len[i] = (int32_t)x.plen;
}

__global__ void edn_write_payload_kernel(const EdnItem* items, int64_t n_items, const EdnOp* op,
                                         const int64_t* contrib, const int64_t* off_incl, int32_t* pl) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k >= n_items || !contrib[k]) return;
    const EdnItem& it = items[k];
    int32_t* w = pl + off_incl[k] - contrib[k];
    const uint8_t pm = op[it.op].pm;
    if (pm == PM_BANK) {
        w[0] = (int32_t)it.id;
        const bool have = it.map_kind == 1 && it.vk[MV_DEBITS] == SK_INT && it.vk[MV_CREDITS] == SK_INT;
        w[1] = have ? (int32_t)(it.v[MV_CREDITS] - it.v[MV_DEBITS]) : JTB_NIL;
    } else if (pm == PM_TRIPLES) {
        int m = 0;
        for (int q = 0; q < 2; ++q) {
            if (it.vk[MV_DEBITS + q] != SK_INT) continue;
            const uint64_t u = (uint64_t)it.v[MV_DEBITS + q];
            w[m++] = (int32_t)(2 * it.id + q);
            w[m++] = (int32_t)(uint32_t)u;
            w[m++] = (int32_t)(uint32_t)(u >> 32);
        }
    } else {
        const uint64_t u = (uint64_t)it.id;
        w[0] = (int32_t)(uint32_t)u;
        w[1] = (int32_t)(uint32_t)(u >> 32);
        w[2] = (int32_t)it.v[MV_DEBIT];
        w[3] = (int32_t)it.v[MV_CREDIT];
        w[4] = (int32_t)it.v[MV_AMOUNT];
    }
}

template <class Pred>
struct EdnCount {   // a selection predicate as 0 / 1, to size the selection before it is made
    Pred pred;
    template <class T>
    __device__ int64_t operator()(T x) const { return pred(x) ? 1 : 0; }
};

// frees the page-locked arrays of out and clears it
inline void jtb_edn_history_release(jtb_edn_history* out) {
    jtb_history& h = out->history;
    for (void* p : {(void*)h.type, (void*)h.f, (void*)h.flags, (void*)h.process, (void*)h.index, (void*)h.time_ns,
                    (void*)h.a, (void*)h.b, (void*)h.c, (void*)h.payload_off, (void*)h.payload_len, (void*)h.payload,
                    (void*)h.shard_off, (void*)h.key_ids})
        if (p) cudaFreeHost(p);
    std::memset(out, 0, sizeof *out);
}

inline unsigned edn_blocks(int64_t n, int threads = 256) {
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, INT_MAX));
}

// The device state passes 1–5 leave behind, on one call's allocations, and the scratch they share with the passes
// after them (the cub temporary storage grows as a later call needs more).  K18 (`run_read_ledger_edn`) and K19
// (`run_ledger_edn_checks`, jtb_edn_checks.cuh) both start with `edn_parse`.
struct EdnParse {
    cudaStream_t st;
    CallAllocs& A;
    void* tmp = nullptr;
    size_t tmp_cap = 0, bytes = 0;
    int64_t* d_cnt = nullptr;           // 4 counters for reductions and selections
    char* text = nullptr;               // the text, padded with 64 spaces
    int* depth = nullptr;               // per byte: the bracket depth (an open counts itself)
    int64_t N = 0;                      // max(n, 1)
    unsigned long long* err = nullptr;  // [0] the first error (byte << 8 | EdnErr), [1] multi-transfer txns
    int base = 0;                       // the depth of the op maps (1: one vector of ops)
    uint32_t* lv2 = nullptr;            // the brackets sorted by (level, position): levels ...
    int64_t *br2 = nullptr, nb = 0;     // ... and positions; pairs (2k, 2k + 1) match
    int64_t *forms = nullptr, nf = 0;   // every form start at depth <= the reader's limit
    int64_t *ops = nullptr, n_ops = 0, *ch = nullptr, n_ch = 0, *it_pos = nullptr, n_it = 0;
    int32_t* n_child = nullptr;         // per op: its map's forms
    int32_t* field = nullptr;           // per op and EK_*: the child index of the key's value + 1, 0 absent
    EdnOp* op = nullptr;
    EdnItem* items = nullptr;
    int64_t* contrib = nullptr;
    int32_t *cl = nullptr, *cl2 = nullptr, *key2 = nullptr;   // ledger-lookups: client ops in history order, sorted
    int64_t n_cl = 0;                                         // by (process, position), and their processes
    std::chrono::steady_clock::time_point t_h2d;              // when the text was on the device

    EdnParse(cudaStream_t s, CallAllocs& a) : st(s), A(a) {}

    cudaError_t need_tmp(size_t b) {   // grow the cub temporary storage
        if (b <= tmp_cap) return cudaSuccess;
        char* p;
        const cudaError_t e = A.alloc(&p, b);
        if (e == cudaSuccess) { tmp = p; tmp_cap = b; }
        return e;
    }
    cudaError_t fetch(int64_t* dst, const int64_t* src) {
        cudaError_t e = cudaMemcpyAsync(dst, src, 8, cudaMemcpyDeviceToHost, st);
        return e == cudaSuccess ? cudaStreamSynchronize(st) : e;
    }
    cudaError_t error_word(unsigned long long* w) {
        cudaError_t e = cudaMemcpyAsync(w, err, 8, cudaMemcpyDeviceToHost, st);
        return e == cudaSuccess ? cudaStreamSynchronize(st) : e;
    }
    // how many of in[0, n_in) satisfy pred
    template <class In, class Pred>
    cudaError_t count(In in, int64_t n_in, Pred pred, int64_t* n_out) {
        auto flags_it = thrust::make_transform_iterator(in, EdnCount<Pred>{pred});
        cudaError_t e = cub::DeviceReduce::Sum(nullptr, bytes, flags_it, d_cnt, n_in, st);
        if (e == cudaSuccess) e = need_tmp(bytes);
        if (e == cudaSuccess) e = cub::DeviceReduce::Sum(tmp, bytes, flags_it, d_cnt, n_in, st);
        return e == cudaSuccess ? fetch(n_out, d_cnt) : e;
    }
    // the elements of in[0, n_in) that satisfy pred, in order, into out (sized by count)
    template <class In, class Out, class Pred>
    cudaError_t select_into(In in, int64_t n_in, Pred pred, Out* out) {
        cudaError_t e = cub::DeviceSelect::If(nullptr, bytes, in, out, d_cnt, n_in, pred, st);
        if (e == cudaSuccess) e = need_tmp(bytes);
        return e == cudaSuccess ? cub::DeviceSelect::If(tmp, bytes, in, out, d_cnt, n_in, pred, st) : e;
    }
    // count, then select into a buffer of that size
    template <class In, class Pred>
    cudaError_t select(In in, int64_t n_in, Pred pred, int64_t** outp, int64_t* n_out) {
        cudaError_t e = count(in, n_in, pred, n_out);
        if (e == cudaSuccess) e = A.alloc(outp, (size_t)std::max<int64_t>(*n_out, 1));
        return e == cudaSuccess ? select_into(in, n_in, pred, *outp) : e;
    }
};

// Why the input was refused: a byte position (-1: none) and a reason; reason == nullptr when it was not.
struct EdnRefusal {
    int64_t at = -1;
    const char* reason = nullptr;
    void set(unsigned long long w) { at = (int64_t)(w >> 8); reason = edn_err_text((uint32_t)(w & 0xff)); }
};

// Passes 1–4 on text[0, n), shared by every reader: the text copied to the device (P.t_h2d, then ev0 recorded), string
// state, depth, bracket pairing, the form starts at depth <= max_depth, ops, their map entries and the forms one level
// below those, and where each op's keys are (P.n_child, P.field).  Returns 0 (r.reason set when the input is refused) or
// -1 with err on a CUDA or allocation error.
inline int edn_parse_forms(EdnParse& P, cudaEvent_t ev0, const char* text, int64_t n, int max_depth, EdnRefusal& r,
                           std::string& err) {
    cudaStream_t st = P.st;
    CallAllocs& A = P.A;
    const int T = 256;
    const int64_t N = P.N = std::max<int64_t>(n, 1);
    JTB_OK(A.alloc(&P.text, (size_t)N + 64));
    JTB_OK(A.alloc(&P.err, 2));
    char* d_text = P.text;
    unsigned long long* d_err = P.err;
    JTB_OK(cudaMemsetAsync(d_text, ' ', (size_t)N + 64, st));
    JTB_OK(cudaMemsetAsync(d_err, 0xff, 16, st));
    if (n) JTB_OK(cudaMemcpyAsync(d_text, text, (size_t)n, cudaMemcpyHostToDevice, st));
    JTB_OK(cudaStreamSynchronize(st));
    P.t_h2d = std::chrono::steady_clock::now();
    JTB_OK(cudaEventRecord(ev0, st));
    size_t& bytes = P.bytes;
    unsigned long long w = ~0ull;

    // ---- 1, 2: string state, depth, byte checks, bracket pairing ----------------------------------------------------
    uint8_t* par;
    int* depth;
    JTB_OK(A.alloc(&par, (size_t)N));
    JTB_OK(A.alloc(&depth, (size_t)N));
    P.depth = depth;
    JTB_OK(A.alloc(&P.d_cnt, 4));
    int64_t* d_cnt = P.d_cnt;
    auto cnt = thrust::counting_iterator<int64_t>(0);
    auto quotes = thrust::make_transform_iterator(cnt, EdnQuote{d_text});
    auto deltas = thrust::make_transform_iterator(cnt, EdnDelta{d_text, par});
    JTB_OK(cub::DeviceScan::InclusiveScan(nullptr, bytes, quotes, par, EdnXor{}, N, st));
    JTB_OK(P.need_tmp(bytes));
    JTB_OK(cub::DeviceScan::InclusiveScan(P.tmp, bytes, quotes, par, EdnXor{}, N, st));
    JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, bytes, deltas, depth, N, st));
    JTB_OK(P.need_tmp(bytes));
    JTB_OK(cub::DeviceScan::InclusiveSum(P.tmp, bytes, deltas, depth, N, st));
    edn_byte_check_kernel<<<edn_blocks(N / 4), T, 0, st>>>(d_text, par, depth, N, d_err);
    JTB_OK(cudaGetLastError());
    {
        uint8_t last_par = 0;
        int last_depth = 0;
        JTB_OK(cudaMemcpyAsync(&last_par, par + N - 1, 1, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(&last_depth, depth + N - 1, 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(P.error_word(&w));
        if (w != ~0ull) { r.set(w); return 0; }
        if (last_par) { r.reason = "unterminated string"; return 0; }
        if (last_depth != 0) { r.reason = "unbalanced brackets"; return 0; }
    }
    int64_t* br;
    JTB_OK(P.select(cnt, N, EdnIsBracket{d_text, par}, &br, &P.nb));
    const int64_t nb = P.nb;
    if (nb) {
        uint32_t* lv;
        JTB_OK(A.alloc(&lv, (size_t)nb));
        JTB_OK(A.alloc(&P.lv2, (size_t)nb));
        JTB_OK(A.alloc(&P.br2, (size_t)nb));
        edn_bracket_level_kernel<<<edn_blocks(nb), T, 0, st>>>(d_text, depth, br, nb, lv);
        JTB_OK(cudaGetLastError());
        uint32_t* d_max = (uint32_t*)d_cnt;
        JTB_OK(cub::DeviceReduce::Max(nullptr, bytes, lv, d_max, nb, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceReduce::Max(P.tmp, bytes, lv, d_max, nb, st));
        uint32_t max_level = 0;
        JTB_OK(cudaMemcpyAsync(&max_level, d_max, 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        int end_bit = 1;
        while (end_bit < 32 && (max_level >> end_bit)) ++end_bit;
        JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, lv, P.lv2, br, P.br2, nb, 0, end_bit, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceRadixSort::SortPairs(P.tmp, bytes, lv, P.lv2, br, P.br2, nb, 0, end_bit, st));
        edn_bracket_pair_kernel<<<edn_blocks((nb + 1) / 2), T, 0, st>>>(d_text, P.lv2, P.br2, nb, d_err);
        JTB_OK(cudaGetLastError());
        JTB_OK(P.error_word(&w));
        if (w != ~0ull) { r.set(w); return 0; }
    }

    // ---- 3: form starts, the base depth, ops, their children and micro-ops ------------------------------------------
    JTB_OK(P.select(cnt, N, EdnFormStart{d_text, par, depth, max_depth}, &P.forms, &P.nf));
    const int64_t* forms = P.forms;
    const int64_t nf = P.nf;
    int base = 0;
    if (nf) {
        int* d_top = (int*)d_cnt;
        JTB_OK(cudaMemsetAsync(d_top, 0, 4, st));
        edn_top_kernel<<<edn_blocks(nf), T, 0, st>>>(d_text, depth, forms, nf, d_top);
        JTB_OK(cudaGetLastError());
        int n_top = 0;
        int64_t first = 0;
        char first_c = 0, before = 0;
        JTB_OK(cudaMemcpyAsync(&n_top, d_top, 4, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaMemcpyAsync(&first, forms, 8, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        JTB_OK(cudaMemcpyAsync(&first_c, d_text + first, 1, cudaMemcpyDeviceToHost, st));
        if (first > 0) JTB_OK(cudaMemcpyAsync(&before, d_text + first - 1, 1, cudaMemcpyDeviceToHost, st));
        JTB_OK(cudaStreamSynchronize(st));
        if (n_top == 1 && (first_c == '[' || first_c == '(') && before != '#') base = 1;   // one vector of ops
    }
    P.base = base;
    JTB_OK(P.select(forms, nf, EdnAtDepth{d_text, depth, base}, &P.ops, &P.n_ops));
    JTB_OK(P.select(forms, nf, EdnAtDepth{d_text, depth, base + 1}, &P.ch, &P.n_ch));
    JTB_OK(P.select(forms, nf, EdnAtDepth{d_text, depth, base + 2}, &P.it_pos, &P.n_it));
    const int64_t *ops = P.ops, *ch = P.ch;
    const int64_t n_ops = P.n_ops, n_ch = P.n_ch, n_it = P.n_it;
    if (n_ops >= INT_MAX || n_ch >= INT_MAX - 2 || n_it >= INT_MAX) {
        r.reason = "more than 2^31 - 3 ops, map entries or micro-ops";
        return 0;
    }

    // ---- 4: op keys ---------------------------------------------------------------------------------------------------
    int32_t *ch_op, *first_child;
    JTB_OK(A.alloc(&ch_op, (size_t)n_ch));
    JTB_OK(A.alloc(&first_child, (size_t)n_ops));
    JTB_OK(A.alloc(&P.n_child, (size_t)n_ops));
    JTB_OK(A.alloc(&P.field, (size_t)n_ops * EK_N));
    JTB_OK(A.alloc(&P.op, (size_t)n_ops));
    JTB_OK(cudaMemsetAsync(first_child, 0x7f, (size_t)n_ops * 4, st));
    JTB_OK(cudaMemsetAsync(P.n_child, 0, (size_t)n_ops * 4, st));
    JTB_OK(cudaMemsetAsync(P.field, 0, (size_t)n_ops * EK_N * 4, st));
    if (n_ops && n_ch) {
        edn_child_kernel<<<edn_blocks(n_ch), T, 0, st>>>(ops, n_ops, ch, n_ch, ch_op, first_child, P.n_child);
        edn_key_kernel<<<edn_blocks(n_ch), T, 0, st>>>(d_text, ch, n_ch, ch_op, first_child, P.field);
        JTB_OK(cudaGetLastError());
    }
    return 0;
}

// Passes 1–5 on text[0, n) read as `form`: edn_parse_forms (form starts at depth <= 3), then the op fields, micro-ops,
// tags, the per-process sort (ledger-lookups), and the events' and payload's checks.  Returns 0 (r.reason set when the
// input is refused: the first error in the file) or -1 with err on a CUDA or allocation error.
inline int edn_parse(EdnParse& P, cudaEvent_t ev0, const char* text, int64_t n, int32_t form, EdnRefusal& r,
                     std::string& err) {
    if (edn_parse_forms(P, ev0, text, n, 3, r, err) != 0) return -1;
    if (r.reason) return 0;
    cudaStream_t st = P.st;
    CallAllocs& A = P.A;
    const int T = 256;
    const int64_t N = P.N;
    char* d_text = P.text;
    unsigned long long* d_err = P.err;
    int64_t* d_cnt = P.d_cnt;
    size_t& bytes = P.bytes;
    unsigned long long w = ~0ull;
    const int64_t *ops = P.ops, *ch = P.ch, *it_pos = P.it_pos;
    const int64_t n_ops = P.n_ops, n_ch = P.n_ch, n_it = P.n_it;
    int32_t* field = P.field;
    EdnOp* op = P.op;

    // ---- 4: op fields ---------------------------------------------------------------------------------------------
    unsigned long long* d_multi = d_err + 1;
    JTB_OK(cudaMemsetAsync(d_multi, 0, 8, st));
    if (n_ops) {
        edn_op_kernel<<<edn_blocks(n_ops), T, 0, st>>>(d_text, N, ops, n_ops, ch, P.n_child, field, op, d_err);
        JTB_OK(cudaGetLastError());
    }

    // ---- 5: micro-ops, tags, pending tags, payload --------------------------------------------------------------------
    JTB_OK(A.alloc(&P.items, (size_t)n_it));
    JTB_OK(A.alloc(&P.contrib, (size_t)n_it));
    EdnItem* items = P.items;
    if (n_ops) {
        if (n_it)
            edn_item_kernel<<<edn_blocks(n_it), T, 0, st>>>(d_text, N, ops, n_ops, ch, n_ch, it_pos, n_it, op, items,
                                                            d_err);
        edn_tag_kernel<<<edn_blocks(n_ops), T, 0, st>>>(ops, n_ops, op, items, it_pos, form, d_err);
        JTB_OK(cudaGetLastError());
    }
    if (form == JTB_FORM_LEDGER_LOOKUPS && n_ops) {
        int64_t* d_ncl = d_cnt + 1;
        int32_t *key;
        JTB_OK(A.alloc(&P.cl, (size_t)n_ops));
        JTB_OK(A.alloc(&P.cl2, (size_t)n_ops));
        JTB_OK(A.alloc(&key, (size_t)n_ops));
        JTB_OK(A.alloc(&P.key2, (size_t)n_ops));
        auto ci = thrust::counting_iterator<int32_t>(0);
        JTB_OK(cub::DeviceSelect::If(nullptr, bytes, ci, P.cl, d_ncl, n_ops, EdnIsClient{op}, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceSelect::If(P.tmp, bytes, ci, P.cl, d_ncl, n_ops, EdnIsClient{op}, st));
        JTB_OK(P.fetch(&P.n_cl, d_ncl));
        const int64_t n_cl = P.n_cl;
        if (n_cl) {
            edn_proc_key_kernel<<<edn_blocks(n_cl), T, 0, st>>>(op, P.cl, n_cl, key);
            JTB_OK(cudaGetLastError());
            JTB_OK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, key, P.key2, P.cl, P.cl2, n_cl, 0, 32, st));
            JTB_OK(P.need_tmp(bytes));
            JTB_OK(cub::DeviceRadixSort::SortPairs(P.tmp, bytes, key, P.key2, P.cl, P.cl2, n_cl, 0, 32, st));
            edn_pending_kernel<<<edn_blocks(n_cl), T, 0, st>>>(ops, op, P.key2, P.cl2, n_cl, d_err);
            JTB_OK(cudaGetLastError());
        }
    }
    if (n_ops) {
        edn_event_kernel<<<edn_blocks(n_ops), T, 0, st>>>(ops, n_ops, op, items, it_pos, form, d_err, d_multi);
        if (n_it) edn_contrib_kernel<<<edn_blocks(n_it), T, 0, st>>>(it_pos, items, n_it, op, P.contrib, d_err);
        JTB_OK(cudaGetLastError());
    }
    JTB_OK(P.error_word(&w));
    if (w != ~0ull) r.set(w);
    return 0;
}

// the host side of jtb_read_ledger_edn
inline int run_read_ledger_edn(cudaStream_t st, cudaEvent_t ev0, cudaEvent_t ev1, const char* text, int64_t n,
                               int32_t form, int32_t flags, jtb_edn_history* out, std::string& err) {
    using Clock = std::chrono::steady_clock;
    const auto t0 = Clock::now();
    if (!out || n < 0 || (n > 0 && !text)) return input_error(err, "malformed arguments");
    if (flags != 0) return input_error(err, "flags must be 0");
    if (form != JTB_FORM_BANK && form != JTB_FORM_LEDGER_COUNTERS && form != JTB_FORM_LEDGER_LOOKUPS)
        return input_error(err, "unknown form %d", (int)form);
    std::memset(out, 0, sizeof *out);
    const int T = 256;
    CallAllocs A;
    EdnParse P(st, A);
    EdnRefusal r;
    if (edn_parse(P, ev0, text, n, form, r, err) != 0) return -1;
    if (r.reason) {
        if (r.at >= 0) return input_error(err, "history.edn at byte %lld: %s", (long long)r.at, r.reason);
        return input_error(err, "history.edn: %s", r.reason);
    }
    const auto t1 = P.t_h2d;
    size_t& bytes = P.bytes;
    const int64_t n_ops = P.n_ops, n_it = P.n_it;
    EdnOp* op = P.op;
    EdnItem* items = P.items;
    int64_t* contrib = P.contrib;
    unsigned long long* d_multi = P.err + 1;

    int64_t *ev_incl, *poff_incl, *it_incl, n_events = 0, n_payload = 0;
    JTB_OK(A.alloc(&ev_incl, (size_t)n_ops));
    JTB_OK(A.alloc(&poff_incl, (size_t)n_ops));
    JTB_OK(A.alloc(&it_incl, (size_t)n_it));
    if (n_ops) {
        auto oi = thrust::counting_iterator<int64_t>(0);
        auto keep = thrust::make_transform_iterator(oi, EdnKeep{op});
        auto plen = thrust::make_transform_iterator(oi, EdnPlen{op});
        JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, bytes, keep, ev_incl, n_ops, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceScan::InclusiveSum(P.tmp, bytes, keep, ev_incl, n_ops, st));
        JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, bytes, plen, poff_incl, n_ops, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceScan::InclusiveSum(P.tmp, bytes, plen, poff_incl, n_ops, st));
        JTB_OK(P.fetch(&n_events, ev_incl + n_ops - 1));
        JTB_OK(P.fetch(&n_payload, poff_incl + n_ops - 1));
    }
    if (n_it) {
        JTB_OK(cub::DeviceScan::InclusiveSum(nullptr, bytes, contrib, it_incl, n_it, st));
        JTB_OK(P.need_tmp(bytes));
        JTB_OK(cub::DeviceScan::InclusiveSum(P.tmp, bytes, contrib, it_incl, n_it, st));
    }
    EdnEvents e;
    int32_t* d_pl;
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
    JTB_OK(A.alloc(&d_pl, (size_t)n_payload));
    if (n_events) {
        edn_write_events_kernel<<<edn_blocks(n_ops), T, 0, st>>>(op, n_ops, ev_incl, poff_incl, e);
        if (n_it) edn_write_payload_kernel<<<edn_blocks(n_it), T, 0, st>>>(items, n_it, op, contrib, it_incl, d_pl);
        JTB_OK(cudaGetLastError());
    }
    unsigned long long multi = 0;
    JTB_OK(cudaMemcpyAsync(&multi, d_multi, 8, cudaMemcpyDeviceToHost, st));
    JTB_OK(cudaEventRecord(ev1, st));
    JTB_OK(cudaStreamSynchronize(st));
    const auto t2 = Clock::now();
    float ms = 0;
    JTB_OK(cudaEventElapsedTime(&ms, ev0, ev1));

    // ---- the arrays, copied into page-locked host memory the library owns ---------------------------------------------
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
    host((void**)&h.shard_off, 16);
    host((void**)&h.key_ids, 8);
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
                                    {(void*)h.payload, d_pl, (size_t)n_payload * 4}})
        if (ce == cudaSuccess) ce = d2h(dst, src, nbytes);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) {
        jtb_edn_history_release(out);
        err = std::string("copying the history back: ") + cudaGetErrorString(ce);
        return -1;
    }
    h.n_events = n_events;
    h.n_payload = n_payload;
    h.n_shards = 1;
    ((int64_t*)h.shard_off)[0] = 0;
    ((int64_t*)h.shard_off)[1] = n_events;
    ((int64_t*)h.key_ids)[0] = -1;
    out->multi_transfer_txns = (int64_t)multi;
    out->n_ops = n_ops;
    const auto t3 = Clock::now();
    out->seconds_h2d = std::chrono::duration<double>(t1 - t0).count();
    out->seconds_kernel = ms * 1e-3;
    out->seconds_d2h = std::chrono::duration<double>(t3 - t2).count();
    out->seconds_total = std::chrono::duration<double>(t3 - t0).count();
    return 0;
}
}  // namespace jtb
