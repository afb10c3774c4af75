/*
 * jtb_check.h — C ABI of the H100-native history checker (libjtb_check.so).
 *
 * This is the drop-in boundary for the ONE hot path of nurturenature/jepsen-tigerbeetle that this
 * repo accelerates: the history checkers that sit behind the Clojure protocol
 * `jepsen.checker/Checker` (`(check [this test history opts]) -> {:valid? ...}`), composed by the
 * reference at
 *     src/tigerbeetle/workloads/set_full.clj:155-158   (independent/checker ∘ compose{set-full, read-all-invoked-adds})
 *     src/tigerbeetle/tests/ledger.clj:363-367         (compose{:SI checker, ...})
 *     src/tigerbeetle/core.clj:139-146                 (top-level compose)
 *
 * A JVM host (JNI) or any FFI binds exactly these entry points; all arguments are plain pointers and
 * sizes owned by the caller for the duration of the call.  Nothing here is a torch type.
 *
 * Verdict coding follows jepsen.checker/merge-valid (false dominates :unknown dominates true):
 *     JTB_VALID (0) < JTB_UNKNOWN (1) < JTB_INVALID (2)   so that merging == max.
 */
#ifndef JTB_CHECK_H
#define JTB_CHECK_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JTB_ABI_VERSION 10

/* ---- verdict lattice (jepsen.checker/merge-valid) ------------------------------------------- */
#define JTB_VALID   0
#define JTB_UNKNOWN 1
#define JTB_INVALID 2

/* ---- op :type (knossos.op/{invoke?,ok?,fail?,info?}) ----------------------------------------- */
#define JTB_T_INVOKE 0
#define JTB_T_OK     1
#define JTB_T_FAIL   2
#define JTB_T_INFO   3

/* ---- op :f opcodes ----------------------------------------------------------------------------
 * register / cas-register (knossos.model):  READ a=value|JTB_NIL ; WRITE a=value ; CAS a=old b=new
 * set (knossos.model/set, jepsen.checker/set-full; set_full.clj:29-31,128-134):
 *                                           ADD a=element ; READ payload=element ids
 * bank (tests/ledger.clj:89-114 after ledger->bank):
 *                                           TRANSFER a=amount b=debit-acct c=credit-acct ;
 *                                           READ payload=(account id, balance) pairs
 */
#define JTB_F_READ     0
#define JTB_F_WRITE    1
#define JTB_F_CAS      2
#define JTB_F_ADD      3
#define JTB_F_TRANSFER 4
#define JTB_F_LOOKUP   5 /* ledger-lookups form only: a [:l-t ...] txn (tigerbeetle.clj:195-213); the :ok payload is the
                            returned transfer records, 5 int32 each (id_lo, id_hi, debit, credit, amount) */

#define JTB_NIL INT32_MIN /* Clojure nil in an int32 field (a nil register read matches any state) */

/* ---- op flags --------------------------------------------------------------------------------- */
#define JTB_FLAG_FINAL 1u /* :final? true  (set_full.clj:45, tests/ledger.clj:78,84) */

/* ---- models for the linearizability search ---------------------------------------------------- */
#define JTB_MODEL_REGISTER     0 /* knossos.model/register      */
#define JTB_MODEL_CAS_REGISTER 1 /* knossos.model/cas-register  */
#define JTB_MODEL_SET          2 /* knossos.model/set (grow-only) */
#define JTB_MODEL_BANK         3 /* bank-transfer model implied by tests/ledger.clj:89-152 */

#define JTB_MAX_ACCOUNTS 8 /* core.clj:208-210 default (vec (range 1 9)) */

/*
 * Flattened history, struct-of-arrays, little-endian, events in history (:index) order.
 * Independent keys (jepsen.independent tuples, set_full.clj:31,44,116,134) are a CSR partition:
 * shard s owns events [shard_off[s], shard_off[s+1]); inside a shard events keep history order.
 * A history without independent keys has n_shards = 1, shard_off = {0, n_events}.
 * Events of non-client processes (:nemesis) carry process < 0 and are ignored by every checker
 * (tests/ledger.clj:94,204,228,262).
 */
typedef struct jtb_history {
    int64_t n_events;
    const uint8_t*  type;        /* [n_events] JTB_T_*                                              */
    const uint8_t*  f;           /* [n_events] JTB_F_*                                              */
    const uint8_t*  flags;       /* [n_events] JTB_FLAG_* (may be NULL = all zero)                  */
    const int32_t*  process;     /* [n_events] :process, <0 = not a client                          */
    const int32_t*  index;       /* [n_events] original :index (reported back as witness)           */
    const int64_t*  time_ns;     /* [n_events] :time                                                */
    const int32_t*  a;           /* [n_events] see opcodes                                          */
    const int32_t*  b;           /* [n_events]                                                      */
    const int32_t*  c;           /* [n_events]                                                      */
    const int64_t*  payload_off; /* [n_events] offset into payload (in int32 units)                 */
    const int32_t*  payload_len; /* [n_events] number of int32 in this event's payload, -1 = nil    */
    const int32_t*  payload;     /* [n_payload]                                                     */
    int64_t n_payload;
    int32_t n_shards;
    const int64_t*  shard_off;   /* [n_shards+1]                                                    */
    const int64_t*  key_ids;     /* [n_shards] the independent key of each shard (may be NULL)      */
} jtb_history;

typedef struct jtb_model {
    int32_t kind;                         /* JTB_MODEL_*                                            */
    int32_t init_value;                   /* register / cas-register initial value (JTB_NIL = nil)  */
    int32_t n_accounts;                   /* bank: (count (:accounts test)) <= JTB_MAX_ACCOUNTS     */
    int32_t account_ids[JTB_MAX_ACCOUNTS];/* bank: (:accounts test), core.clj:208-210               */
    int32_t init_balance[JTB_MAX_ACCOUNTS];/* bank: starting balances (db.clj:118-127 => zeros)     */
    int32_t negative_balances_ok;         /* bank: (:negative-balances? test), core.clj:217-219     */
} jtb_model;

/* By default the search linearizes a consistent candidate READ immediately and exclusively ("eager
 * reads": a read never changes the model state, so verdict and witness are unchanged while the number
 * of configurations drops by an order of magnitude).  Knossos does not do this; set this flag to visit
 * exactly the configurations Knossos' WGL would. */
#define JTB_OPT_NO_EAGER_READS 1
/* For histories with crashed (:info) ops a few depth-first "scout" warps walk the same configuration space in
 * knossos.wgl's order (and three other orders) beside the exhaustive search, each with a private visited table;
 * a scout can only ever report VALID (it found a linearization), so verdicts, witnesses and exhaustive
 * configuration counts are unaffected.  Set this flag to run the exhaustive search alone. */
#define JTB_OPT_NO_SCOUTS 2
/* Engine choice for jtb_check_linearizable.  Default (neither bit): the level-synchronous engine (csrc/jtb_level.cuh:
 * breadth-first by depth, visited set local to a level, bounded memory) for histories without crashed (:info) ops
 * that are searched in the Knossos-exact space or are wide (nearly every client always has an op in flight), the
 * work-list engine (csrc/jtb_wgl.cuh: depth-first locally, persistent visited table, scouts) otherwise.
 * Verdict, witness and exhaustive configuration counts are identical; the bits force one engine. */
#define JTB_OPT_ENGINE_LEVEL    4
#define JTB_OPT_ENGINE_WORKLIST 8
/* A single-key history with crashed (:info) ops first gets a budgeted run of the work list (16 M configurations) and,
 * if that leaves it open, a BEAM (the level engine expanding only the best ~256, then ~2k, then ~16k configurations of
 * every level: fewest crashed ops consumed, furthest frontier): it finds the linearization of a valid history in tens of
 * milliseconds where an exhaustive search drowns.  A beam can only ever report VALID; what it does not decide goes to
 * the exhaustive search.  Set this flag to skip both. */
#define JTB_OPT_NO_BEAM         16

/* Options for a context.  Zero-initialise, then set what you need. */
typedef struct jtb_opts {
    int32_t  device;            /* CUDA device ordinal for this context                              */
    int32_t  flags;             /* JTB_OPT_* bits                                                     */
    uint64_t table_bytes;       /* visited-config table size in HBM (0 = default 4 GiB)              */
    uint64_t max_configs;       /* search budget: stop with JTB_UNKNOWN after this many (0 = table)   */
    uint32_t time_budget_ms;    /* 0 = unlimited                                                      */
    uint32_t search_ctas;       /* 0 = one persistent CTA per SM × resident CTAs                      */
} jtb_opts;

/* Per-shard output of the linearizability search (knossos analysis map, SURVEY A.5/A.6). */
typedef struct jtb_lin_shard {
    int32_t  valid;             /* JTB_VALID / JTB_UNKNOWN / JTB_INVALID                              */
    int32_t  witness_index;     /* :index of the :ok completion that cannot be linearized (:op), -1   */
    int32_t  previous_ok_index; /* :index of the last :ok completion before it (:previous-ok), -1     */
    int32_t  cause;             /* JTB_CAUSE_* when valid == JTB_UNKNOWN                              */
    uint64_t configs_explored;  /* distinct (linearized-set, model-state) configs inserted            */
    uint64_t probes;            /* visited-table probes (hits + misses)                               */
} jtb_lin_shard;

#define JTB_CAUSE_NONE          0
#define JTB_CAUSE_TABLE_FULL    1 /* visited table exhausted (knossos: out of memory -> :unknown)    */
#define JTB_CAUSE_BUDGET        2 /* max_configs / time budget reached                                */
#define JTB_CAUSE_TOO_WIDE      3 /* > 64 concurrently open completed ops, or key does not fit        */
#define JTB_CAUSE_PARTIAL_READ  4 /* monotonic-key check: an :ok read does not observe every key of its shard */
#define JTB_CAUSE_ANOMALY       5 /* serial-witness check: the transfer-placement check found KEY, JOINT, DOUBLE or LOST */
#define JTB_CAUSE_UNDECIDED     6 /* serial-witness check: the transfer-placement check left a gap undecided          */
#define JTB_CAUSE_NO_WITNESS    7 /* serial-witness check: a witness round did not explain a gap, or max_rounds ran out */
#define JTB_CAUSE_REAL_TIME     8 /* serial-witness check: the serial order of the chosen gaps breaks real time       */
#define JTB_CAUSE_LOOKUP        9 /* lookup witness: an :ok lookup has no place in the serial order of a proved shard   */

typedef struct jtb_lin_result {
    int32_t  valid;             /* merge-valid over shards                                            */
    int32_t  n_failures;        /* number of shards whose verdict is not JTB_VALID (:failures)        */
    uint64_t configs_explored;  /* sum over shards                                                    */
    uint64_t probes;            /* sum over shards                                                    */
    uint64_t hbm_bytes_algorithmic; /* key_bytes*(probes + inserts), SURVEY §8(d)                     */
    uint32_t key_bytes;         /* bytes per visited-table slot used by this call (16/32/64)          */
    uint32_t reserved0;
    double   seconds_kernel;    /* device time of the search kernels (CUDA events)                    */
    double   seconds_total;     /* host wall time of the call incl. flatten-prep, H2D, D2H            */
} jtb_lin_result;

/* Per-shard output of jepsen.checker/set-full (SURVEY A.3). Element lists are returned through
 * caller-provided buffers in jtb_setfull_out. */
typedef struct jtb_setfull_shard {
    int32_t valid;
    int32_t attempt_count, stable_count, lost_count, never_read_count, stale_count, duplicated_count;
    int32_t suspect_final_reads;   /* read-all-invoked-adds: :final? :ok reads missing an invoked add   */
    int64_t stable_latency_max_ms; /* max stable-latency (0 if none)  */
    int64_t lost_latency_max_ms;   /* max lost-latency (0 if none)    */
} jtb_setfull_shard;

/* Per-element classification codes written to jtb_setfull_out.elem_outcome */
#define JTB_SF_NEVER_READ 0
#define JTB_SF_STABLE     1
#define JTB_SF_LOST       2

typedef struct jtb_setfull_out {
    jtb_setfull_shard* shards;     /* [n_shards] required                                             */
    /* optional per-element detail, CSR by shard over tracked elements in first-add-invoke order:     */
    int64_t  elem_capacity;        /* capacity of the arrays below (0 = not wanted)                   */
    int64_t* elem_off;             /* [n_shards+1]                                                    */
    int32_t* elem_id;              /* element value                                                   */
    uint8_t* elem_outcome;         /* JTB_SF_*                                                        */
    int64_t* elem_latency_ms;      /* stable-latency / lost-latency in ms (0 for never-read)          */
    int32_t* elem_dup_count;       /* max multiplicity seen in one read if > 1, else 0                */
    int32_t  valid;                /* merge-valid over shards                                          */
    int32_t  n_failures;
    double   seconds_kernel;
    double   seconds_total;
    /* (read-all-invoked-adds), workloads/set_full.clj:51-75, evaluated in the same pass: every
     * :final? :ok read must contain every :add value ever invoked in its sub-history.  Optional detail
     * (CSR: suspect read -> missing element ids), caller-allocated:                                   */
    int64_t  suspect_capacity;     /* capacity of suspect_shard / suspect_index (0 = not wanted)       */
    int32_t* suspect_shard;
    int32_t* suspect_index;        /* :index of the suspect final read                                 */
    int64_t* suspect_missing_off;  /* [suspect_capacity + 1]                                           */
    int64_t  missing_capacity;
    int32_t* missing_ids;
    int64_t  n_suspect;            /* out: total suspect final reads                                   */
    int32_t  raia_valid;           /* out: JTB_VALID or JTB_INVALID                                    */
    int32_t  reserved1;
} jtb_setfull_out;

/* bank SI checker (tests/ledger.clj:127-192) error classes, in `cond` precedence order */
#define JTB_BANK_OK             0
#define JTB_BANK_UNEXPECTED_KEY 1
#define JTB_BANK_NIL_BALANCE    2
#define JTB_BANK_WRONG_TOTAL    3
#define JTB_BANK_NEGATIVE_VALUE 4

typedef struct jtb_bank_result {
    int32_t valid;                 /* JTB_UNKNOWN when reference_throws (what check-safe makes of the exception) */
    int32_t reference_throws;      /* 1: the reference checker THROWS on this history — err-badness divides by
                                      (:total-amount test) (tests/ledger.clj:122-123), the default is 0
                                      (tests/ledger.clj:356), and util/max-by calls it as soon as one error type has
                                      >= 2 :wrong-total errors; jepsen's check-safe turns that into
                                      {:valid? :unknown}.  All counts / firsts / lasts below are still filled;
                                      :worst then ranks :wrong-total errors by |total - total-amount|.            */
    int64_t read_count;            /* :read-count  */
    int64_t error_count;           /* :error-count */
    int32_t first_error_index;     /* :index of (:op :first-error), -1                                 */
    int32_t first_error_type;      /* JTB_BANK_*                                                        */
    int64_t count_by_type[5];      /* (:count (errors type))                                            */
    int32_t first_index_by_type[5];/* :index of :first                                                  */
    int32_t last_index_by_type[5]; /* :index of :last                                                   */
    int32_t worst_index_by_type[5];/* :index of :worst (err-badness, tests/ledger.clj:116-125)          */
    int64_t lowest_total, highest_total;       /* :wrong-total :lowest / :highest totals                */
    int32_t lowest_index, highest_index;
    double  seconds_kernel;
    double  seconds_total;
} jtb_bank_result;

/* ---- monotonic-key check (Elle's monotonic-key graph, src/tigerbeetle/elle/core.clj) ------------------------------
 * Nodes are the :ok reads (process >= 0, f == JTB_F_READ, type == JTB_T_OK, payload_len >= 0).  A read's payload is
 * (key:int32, value_lo:int32, value_hi:int32) triples, value = int64 of any sign; for ledger histories key = 2*account
 * + field, field 0 = debits-posted, 1 = credits-posted (counters that only grow), so with accounts in [0, 2^30) every
 * key lies in [0, INT32_MAX].  Reads are ordered by the sum of their values, taken in 128 bits.  Edges:
 *   monotonic  r -> s  when v_k(r) < v_k(s) for some key k both read
 *   real-time  r -> s  when r's completion precedes s's invocation (the latest invoke of s's process before s
 *                      completes; off with JTB_MONO_NO_REALTIME)
 * A shard is JTB_INVALID when the graph has a cycle.  A shard in which some :ok read does not observe every key of
 * the shard is JTB_UNKNOWN with JTB_CAUSE_PARTIAL_READ.  DESIGN.md "K7 monotonic-key check". */
#define JTB_MONO_NO_REALTIME 1

#define JTB_MONO_EDGE_NONE      0
#define JTB_MONO_EDGE_MONOTONIC 1 /* edge_key = key, edge_value = v_key(source), edge_value2 = v_key(target)      */
#define JTB_MONO_EDGE_REALTIME  2 /* edge_key = -1, edge_value = :index of the source's completion,
                                     edge_value2 = :index of the target's invocation                             */

typedef struct jtb_mono_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN / JTB_INVALID                                          */
    int32_t cause;              /* JTB_CAUSE_* when valid == JTB_UNKNOWN                                          */
    int32_t n_reads;            /* :ok reads (graph nodes) of the shard                                           */
    int32_t n_keys;             /* distinct keys the shard's :ok reads observe                                    */
    int32_t witness_index;      /* :index of the earliest :ok read completion whose prefix has a cycle, -1        */
    int32_t partner_index;      /* smallest completion :index of a read forming a 2-cycle with the witness, -1    */
    int32_t edge_kind[2];       /* [0] partner -> witness, [1] witness -> partner: JTB_MONO_EDGE_*                */
    int32_t edge_key[2];
    int64_t edge_value[2];
    int64_t edge_value2[2];
} jtb_mono_shard;

typedef struct jtb_mono_result {
    int32_t valid;              /* merge-valid over shards                                                         */
    int32_t n_failures;         /* shards whose verdict is not JTB_VALID                                           */
    int64_t n_reads;            /* :ok reads over all shards                                                       */
    double  seconds_kernel;     /* device time (CUDA events)                                                       */
    double  seconds_total;      /* host wall time of the call incl. the host pass, H2D, D2H                        */
} jtb_mono_result;

/* ---- counter-bounds check (DESIGN.md "K8 counter-bounds check") ------------------------------------------------------
 * The same reads as the monotonic-key check (:ok, f == JTB_F_READ, (key, value_lo, value_hi) triples, key =
 * 2*account + field).  A transfer is an invoke with f == JTB_F_TRANSFER, a = amount, b = debit account, c = credit
 * account (amounts int32 >= 0, accounts in [0, 2^30)); its fate is the next event of its process (:ok, :info, :fail,
 * or none).  It adds `a` to key 2b+0
 * (debits-posted) and to key 2c+1 (credits-posted); :fail transfers add nothing.  Positions are event positions in the
 * shard.  Counters start at zero and only grow, so under strict serializability every key k an :ok read r observes
 * satisfies L_k(r) <= v_k(r) <= U_k(r):
 *   L = the amounts of the :ok transfers on k that completed before r was invoked (0 when r has no invocation)
 *   U = the amounts of the non-:fail transfers on k invoked before r completed
 * A shard with some (read, key) outside [L, U] is JTB_INVALID, every other shard JTB_VALID. */
#define JTB_CB_BELOW 1 /* v < L: a completed :ok transfer is missing from the read (value = v, bound = L)               */
#define JTB_CB_ABOVE 2 /* v > U: the read holds more than every transfer invoked before it completed (bound = U)        */

typedef struct jtb_cb_shard {
    int32_t valid;              /* JTB_VALID / JTB_INVALID                                                            */
    int32_t n_reads;            /* :ok reads of the shard                                                             */
    int32_t n_transfers;        /* transfers of the shard whose fate is not :fail                                     */
    int32_t n_keys;             /* distinct keys the shard's :ok reads observe                                        */
    int64_t n_below;            /* (read, key) pairs with v < L                                                       */
    int64_t n_above;            /* (read, key) pairs with v > U                                                       */
    int32_t witness_index;      /* :index of the earliest-completing :ok read with a key out of bounds, -1            */
    int32_t witness_key;        /* its smallest such key, -1                                                          */
    int32_t kind;               /* JTB_CB_BELOW / JTB_CB_ABOVE, 0 when VALID                                          */
    int32_t culprit_index;      /* BELOW: completion :index of the first transfer, in completion order, at which the
                                   running sum of L's amounts exceeds value; ABOVE: invocation :index of the last
                                   transfer counted in U (-1 when none)                                                */
    int64_t value;              /* the witness read's value of witness_key                                            */
    int64_t bound;              /* the bound it violates (L for BELOW, U for ABOVE)                                   */
} jtb_cb_shard;

typedef struct jtb_cb_result {
    int32_t valid;              /* merge-valid over shards                                                            */
    int32_t n_failures;         /* INVALID shards                                                                     */
    int64_t n_reads;            /* :ok reads over all shards                                                          */
    int64_t n_transfers;        /* non-:fail transfers over all shards                                                */
    int64_t n_violations;       /* out-of-bounds (read, key) pairs over all shards                                    */
    double  seconds_kernel;     /* device time (CUDA events)                                                          */
    double  seconds_total;      /* host wall time of the call incl. the host pass, H2D, D2H                           */
} jtb_cb_result;

/* ---- transfer-lookup check (DESIGN.md "K9 transfer-lookup check") ----------------------------------------------------
 * Input: the ledger-lookups form.  Reads are the monotonic-key check's.  A transfer invoke (f == JTB_F_TRANSFER) carries
 * one 5-int32 record (id_lo, id_hi, debit, credit, amount) per [:t ...] micro-op; each is one transfer with the txn's
 * interval and fate (the next event of its process).  A lookup is an :ok event with f == JTB_F_LOOKUP whose payload is
 * the returned records in the same layout; its invocation is the latest invoke of its process.  Ids are int64
 * (id_hi << 32 | id_lo) of any sign, ordered as signed integers.  With l an :ok lookup and t a transfer of the same shard, each of these proves an anomaly:
 *   1 PHANTOM            a record whose id no transfer invoke of the shard carries
 *   2 MISMATCH           a record whose (debit, credit, amount) differs from its invocation's
 *   3 FAILED_VISIBLE     a record of a transfer whose fate is :fail
 *   4 FUTURE             a record of a transfer invoked after l completed
 *   5 DUPLICATE          an id twice in one lookup
 *   6 LOST / 7 VANISHED  M(t) = min(t's :ok completion, the earliest completion of an :ok lookup returning t); every
 *                        :ok lookup invoked after M(t) must contain t (LOST when M is the :ok completion)
 *   8 READ_BELOW_LOOKUP  an :ok read's value of key k is below S_k(l) for a lookup l completed before it was invoked
 *   9 READ_ABOVE_LOOKUP  ... above S_k(l) for a lookup l invoked after it completed
 * S_k(l) = the sum over l's distinct ids (first record of each) of the record's amount on k (key 2*debit+0 and
 * 2*credit+1); only keys the shard's :ok reads observe count. */
#define JTB_TL_PHANTOM           1
#define JTB_TL_MISMATCH          2
#define JTB_TL_FAILED_VISIBLE    3
#define JTB_TL_FUTURE            4
#define JTB_TL_DUPLICATE         5
#define JTB_TL_LOST              6
#define JTB_TL_VANISHED          7
#define JTB_TL_READ_BELOW_LOOKUP 8
#define JTB_TL_READ_ABOVE_LOOKUP 9
#define JTB_TL_KINDS             9

typedef struct jtb_tl_shard {
    int32_t valid;              /* JTB_VALID / JTB_INVALID                                                            */
    int32_t n_lookups;          /* :ok lookups of the shard                                                           */
    int64_t n_records;          /* records of those lookups                                                           */
    int32_t n_transfers;        /* transfer micro-ops of the shard (every fate)                                       */
    int32_t n_reads;            /* :ok reads of the shard                                                             */
    int64_t count_by_kind[JTB_TL_KINDS]; /* [kind - 1]: records (1-4), repeated records (5), (lookup, missing
                                   transfer) pairs (6-7), (read, key) pairs (8-9)                                     */
    int32_t witness_index;      /* completion :index of the earliest-completing :ok lookup or read with a violation  */
    int32_t kind;               /* the smallest code among its violations, 0 when VALID                               */
    int64_t transfer_id;        /* lookup kinds: the smallest transfer id of that kind; read kinds: 0                 */
    int32_t key;                /* read kinds: the smallest key of that kind; lookup kinds: -1                        */
    int32_t related_index;      /* LOST: the transfer's completion :index; VANISHED: the earlier lookup's completion
                                   :index; 2-4: the transfer's invocation :index; BELOW: completion :index of the
                                   earliest-completing qualifying lookup with S > value; ABOVE: of the
                                   earliest-invoked qualifying lookup with S < value; PHANTOM, DUPLICATE: -1          */
    int64_t value;              /* read kinds: the read's value of key                                               */
    int64_t bound;              /* read kinds: max S (BELOW) / min S (ABOVE) over the qualifying lookups             */
} jtb_tl_shard;

typedef struct jtb_tl_result {
    int32_t valid;              /* merge-valid over shards                                                            */
    int32_t n_failures;         /* INVALID shards                                                                     */
    int64_t n_lookups;          /* :ok lookups over all shards                                                        */
    int64_t n_records;          /* their records                                                                      */
    int64_t n_transfers;        /* transfer micro-ops                                                                 */
    int64_t n_reads;            /* :ok reads                                                                          */
    int64_t n_violations;       /* sum of count_by_kind over shards and kinds                                         */
    double  seconds_kernel;     /* device time (CUDA events)                                                          */
    double  seconds_total;      /* host wall time of the call incl. the host pass, H2D, D2H                           */
} jtb_tl_result;

/* ---- read-explanation check (DESIGN.md "K10 read-explanation check") -------------------------------------------------
 * Input: the ledger-lookups form, read exactly as the transfer-lookup check reads it.  Every [:t ...] micro-op is one
 * transfer with its txn's interval and fate; it adds its amount to key 2*debit+0 and key 2*credit+1.  With M(t) and the
 * lookups as in K9, and A(t) = the latest invocation of an :ok lookup whose records lack t (-1 when none), every
 * transfer t of the shard of an :ok read r (invocation iv, completion cp) is in exactly one class:
 *   must    M(t) < iv (t was :ok, or returned by an :ok lookup, before r was invoked)
 *   cannot  otherwise, when t's fate is :fail, t was invoked after cp, or A(t) > cp
 *   may     every other transfer with a nonzero amount on a key r observes
 * With d_k = v_k(r) - (the must transfers' sum on k), r is explained when some subset X of its "may" transfers has sum
 * d_k on every key k it observes.  The decision is budgeted, and the budget is deterministic: a read observing more than
 * JTB_RX_MAX_KEYS keys or with more than JTB_RX_MAX_GATHER "may" transfers, one with more than JTB_RX_MAX_FREE of them
 * left after the root pruning, and one whose canonical search visits more than max_nodes nodes are UNDECIDED.  A shard
 * is JTB_INVALID when some read is not explained, else JTB_UNKNOWN when some read is undecided, else JTB_VALID. */
#define JTB_RX_KEY   1 /* some single observed key has no subset of the "may" transfers summing to d_k             */
#define JTB_RX_JOINT 2 /* every key alone has one, but no one subset closes all of them (torn / fractured transfers) */
#define JTB_RX_MAX_KEYS   256
#define JTB_RX_MAX_GATHER 128
#define JTB_RX_MAX_FREE   64
#define JTB_RX_DEFAULT_MAX_NODES 4096 /* max_nodes <= 0 */

typedef struct jtb_rx_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN / JTB_INVALID                                              */
    int32_t n_reads;            /* :ok reads of the shard                                                             */
    int32_t n_transfers;        /* transfer micro-ops of the shard (every fate)                                       */
    int32_t witness_index;      /* completion :index of the earliest-completing unexplained read, -1                  */
    int64_t n_explained;        /* reads explained                                                                    */
    int64_t n_undecided;        /* reads left undecided by the budget                                                 */
    int64_t count_by_kind[2];   /* [kind - 1]: unexplained reads of that kind                                         */
    int64_t nodes;              /* search nodes over the shard's reads, the per-key searches of unexplained reads
                                   included                                                                           */
    int32_t kind;               /* JTB_RX_KEY / JTB_RX_JOINT, 0 when no read is unexplained                           */
    int32_t key;                /* KEY: the smallest key without a subset; JOINT: the smallest key the root pruning
                                   found unreachable, -1 when only the search refuted the read                        */
    int32_t n_must;             /* |must| of the witness read: must transfers on a key it observes                    */
    int32_t n_may;              /* "may" transfers of the witness read the root pruning did not drop                  */
    int64_t value;              /* KEY: the witness read's value of key                                               */
    int64_t must_sum;           /* KEY: the must transfers' sum on key                                                */
} jtb_rx_shard;

typedef struct jtb_rx_result {
    int32_t valid;              /* merge-valid over shards                                                            */
    int32_t n_failures;         /* shards that are not VALID                                                          */
    int64_t n_reads;            /* :ok reads                                                                          */
    int64_t n_transfers;        /* transfer micro-ops                                                                 */
    int64_t n_explained;
    int64_t n_unexplained;
    int64_t n_undecided;
    int64_t nodes;
    double  seconds_kernel;     /* device time (CUDA events)                                                          */
    double  seconds_total;      /* host wall time of the call incl. the host pass, H2D, D2H                           */
} jtb_rx_result;

/* ---- read-gap check (DESIGN.md "K11 read-gap check") ----------------------------------------------------------------
 * Input: the ledger-lookups form, read as the read-explanation check reads it (M(t), A(t) and the fates are K10's).  A
 * shard whose :ok reads do not all observe every key of the shard is JTB_UNKNOWN with JTB_CAUSE_PARTIAL_READ.  On the
 * others the :ok reads are ordered as the monotonic-key check orders them, by (S = the sum of the values, invocation
 * position), r_1 ... r_n, and each read closes one gap: gap 0 from the zero state to r_1, gap i from r_i to r_{i+1},
 * with Delta_k = v_k(r_{i+1}) - v_k(r_i).  A transfer is eligible for gap i unless its fate is :fail, it was invoked
 * after r_{i+1} completed, A(t) > cp(r_{i+1}), or (i >= 1) M(t) < iv(r_i); transfers with a zero amount on every
 * observed key are ignored, and so are those whose amount exceeds Delta_k on one of their keys (no subset summing to
 * Delta holds them).  A gap with some Delta_k < 0 is unexplained (KEY: the two reads form a monotonic-key 2-cycle);
 * Delta = 0 is explained; otherwise the gap is explained when a subset of its eligible transfers sums to Delta_k on
 * every key, decided with the read-explanation check's caps (the gather cap after the amount filter), pruning,
 * canonical search and node budget.
 * A transfer the root pruning forces into two gaps is DOUBLE: the differences between successive read states are
 * disjoint.  A shard is JTB_INVALID when some gap is unexplained or some transfer DOUBLE, else JTB_UNKNOWN when some
 * gap is undecided, else JTB_VALID. */
#define JTB_RG_KEY    1 /* some Delta_k < 0, or some key alone has no subset of the eligible transfers that fit under
                           Delta (amount <= Delta on each of its observed keys) summing to Delta_k                  */
#define JTB_RG_JOINT  2 /* every key alone has one, but no one subset closes all of them                              */
#define JTB_RG_DOUBLE 3 /* a transfer the root pruning forces into this gap and into an earlier one                   */
#define JTB_RG_MAX_KEYS   256
#define JTB_RG_MAX_GATHER 128
#define JTB_RG_MAX_FREE   64
#define JTB_RG_DEFAULT_MAX_NODES 4096 /* max_nodes <= 0 */

typedef struct jtb_rg_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN / JTB_INVALID                                              */
    int32_t cause;              /* JTB_CAUSE_PARTIAL_READ when a partial read makes the shard UNKNOWN, else 0         */
    int32_t n_reads;            /* :ok reads of the shard; a full-key shard has as many gaps                          */
    int32_t n_transfers;        /* transfer micro-ops of the shard (every fate)                                       */
    int64_t n_explained;        /* gaps explained                                                                     */
    int64_t n_undecided;        /* gaps left undecided by the budget                                                  */
    int64_t count_by_kind[3];   /* unexplained gaps of kind KEY, of kind JOINT, and DOUBLE transfers                  */
    int64_t nodes;              /* search nodes over the shard's gaps, the per-key searches of unexplained gaps
                                   included                                                                           */
    int32_t witness_index;      /* completion :index of r_{i+1} of the first violating gap in the order, -1          */
    int32_t lower_index;        /* completion :index of r_i, -1 for gap 0 or no witness                               */
    int32_t kind;               /* JTB_RG_KEY / JOINT / DOUBLE (the smallest at the witness gap), 0 without one       */
    int32_t key;                /* KEY: the smallest refuted key; JOINT: the smallest key the root pruning found
                                   unreachable, -1 when only the search refuted the gap; DOUBLE: -1                   */
    int64_t delta;              /* KEY: Delta_k of key                                                                */
    int64_t transfer_id;        /* DOUBLE: the transfer's id (the smallest at the witness gap)                        */
    int32_t other_index;        /* DOUBLE: completion :index of the upper read of the earlier gap, -1                 */
    int32_t n_eligible;         /* eligible transfers of the witness gap the root pruning did not drop                */
} jtb_rg_shard;

typedef struct jtb_rg_result {
    int32_t valid;              /* merge-valid over shards                                                            */
    int32_t n_failures;         /* shards that are not VALID                                                          */
    int64_t n_reads;            /* :ok reads                                                                          */
    int64_t n_transfers;        /* transfer micro-ops                                                                 */
    int64_t n_explained;        /* gaps explained                                                                     */
    int64_t n_unexplained;      /* gaps unexplained (KEY + JOINT)                                                     */
    int64_t n_double;           /* DOUBLE transfers                                                                   */
    int64_t n_undecided;        /* gaps undecided                                                                     */
    int64_t nodes;
    double  seconds_kernel;     /* device time (CUDA events)                                                          */
    double  seconds_total;      /* host wall time of the call incl. the host pass, H2D, D2H                           */
} jtb_rg_result;

/* ---- transfer-placement check (DESIGN.md "K12 transfer-placement check") --------------------------------------------
 * Input, shards, reads, their order r_1 ... r_n, the gaps, Delta, M(t) and A(t): the read-gap check's.  Every transfer
 * that is not :fail, has a positive amount and touches a key the shard observes gets a window of gaps [lo, hi]: t is in
 * no gap before lo (some read at or before lo in the order completed before t was invoked, or A(t) > its completion),
 * and a "must" transfer (M(t) < the invocation of some read) is in exactly one gap at or before hi, the gap of the first
 * such read; a "may" transfer has hi = the last gap and may lie in none.  Then rounds (Jacobi: each reads only the state
 * the previous one left):
 *   - round 0 is the read-gap check, gap for gap (gather, caps, pruning, search, nodes, DOUBLE);
 *   - after every round, per transfer: one the root pruning forced into exactly one gap this round is owned by it
 *     (into two: DOUBLE); a must transfer with exactly one possible gap (gathered, and not pruned out there) left in its
 *     window is owned by it (PLACE); one with none is LOST.  PLACE and LOST need every gap of the window complete
 *     (not past the gather cap, at most JTB_TP_MAX_KEYS keys);
 *   - round 1 re-runs every gap, round r >= 2 the gaps in the window of a transfer whose owner changed in round r - 1;
 *     a re-run gap uses Delta' = Delta - the amounts of the transfers it owns (a negative component is KEY) and gathers
 *     only the in-window transfers no gap owns;
 *   - the rounds stop after a round r >= 1 that changes no owner, or after max_rounds.
 * Anomalies latch (a gap unexplained in some round stays so, with its first kind).  A shard is JTB_INVALID on an
 * unexplained gap, a DOUBLE or a LOST transfer, else JTB_UNKNOWN when a gap is undecided in the last round that ran it,
 * else JTB_VALID. */
#define JTB_TP_KEY    1 /* a gap with some Delta'_k < 0, or a key alone no subset of the gathered transfers closes    */
#define JTB_TP_JOINT  2 /* every key alone closes, but no one subset closes all of them                               */
#define JTB_TP_DOUBLE 3 /* a transfer the root pruning forces into two gaps in one round                              */
#define JTB_TP_LOST   4 /* a must transfer with no possible gap left in its window                                    */
#define JTB_TP_MAX_KEYS   JTB_RG_MAX_KEYS
#define JTB_TP_MAX_GATHER JTB_RG_MAX_GATHER
#define JTB_TP_MAX_FREE   JTB_RG_MAX_FREE
#define JTB_TP_DEFAULT_MAX_NODES  JTB_RG_DEFAULT_MAX_NODES /* max_nodes <= 0 */
#define JTB_TP_DEFAULT_MAX_ROUNDS 64                       /* max_rounds <= 0 */

typedef struct jtb_tp_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN / JTB_INVALID                                              */
    int32_t cause;              /* JTB_CAUSE_PARTIAL_READ when a partial read makes the shard UNKNOWN, else 0         */
    int32_t n_reads;            /* :ok reads of the shard; a full-key shard has as many gaps                          */
    int32_t n_transfers;        /* transfer micro-ops of the shard (every fate)                                       */
    int64_t n_explained;        /* gaps explained in the last round that ran them and never unexplained               */
    int64_t n_undecided;        /* gaps undecided in the last round that ran them and never unexplained               */
    int64_t count_by_kind[4];   /* unexplained gaps of kind KEY, of kind JOINT, DOUBLE transfers, LOST transfers      */
    int64_t n_placed;           /* transfers owned by a gap at the fixpoint                                           */
    int64_t nodes;              /* search nodes over every round                                                      */
    int32_t rounds;             /* rounds that ran a gap of the shard                                                 */
    int32_t witness_index;      /* completion :index of the read closing the witness gap (LOST: r at hi(t)), -1       */
    int32_t lower_index;        /* completion :index of the read before it in the order, -1                           */
    int32_t kind;               /* JTB_TP_KEY / JOINT / DOUBLE / LOST (the smallest at the witness gap), 0 without one */
    int32_t key;                /* KEY / JOINT: as jtb_rg_shard.key; DOUBLE / LOST: -1                                */
    int32_t round;              /* the round that found the witness, -1 without one                                   */
    int64_t delta;              /* KEY: Delta'_k of key in that round                                                 */
    int64_t transfer_id;        /* DOUBLE / LOST: the transfer's id (the smallest at the witness gap)                 */
    int32_t other_index;        /* DOUBLE: completion :index of the read closing the other gap; LOST: the :index of
                                   the event that fixes M(t); -1                                                      */
    int32_t n_eligible;         /* transfers of the witness gap the root pruning kept in the last round that ran it   */
} jtb_tp_shard;

typedef struct jtb_tp_result {
    int32_t valid;              /* merge-valid over shards                                                            */
    int32_t n_failures;         /* shards that are not VALID                                                          */
    int64_t n_reads;            /* :ok reads                                                                          */
    int64_t n_transfers;        /* transfer micro-ops                                                                 */
    int64_t n_explained;        /* gaps explained                                                                     */
    int64_t n_unexplained;      /* gaps unexplained (KEY + JOINT)                                                     */
    int64_t n_double;           /* DOUBLE transfers                                                                   */
    int64_t n_lost;             /* LOST transfers                                                                     */
    int64_t n_undecided;        /* gaps undecided                                                                     */
    int64_t n_placed;           /* transfers owned at the fixpoint                                                    */
    int64_t nodes;
    int64_t rounds;             /* the most rounds of any shard                                                       */
    double  seconds_kernel;     /* device time (CUDA events)                                                          */
    double  seconds_total;      /* host wall time of the call incl. the host pass, H2D, D2H                           */
} jtb_tp_result;

/* ---- serial-witness check (DESIGN.md "K13 serial-witness check") ---------------------------------------------------
 * Proves a shard linearizable (VALID) or says nothing (UNKNOWN), never INVALID.  It runs the transfer-placement check
 * unchanged (same max_nodes, max_rounds); only a shard that check calls VALID gets a witness, otherwise it is UNKNOWN
 * with cause PARTIAL_READ, ANOMALY (KEY, JOINT, DOUBLE or LOST) or UNDECIDED.  Then:
 *   - witness rounds (Jacobi): every gap g whose Delta' (Delta minus the transfers g owns) is not zero gathers as a
 *     transfer-placement round >= 1 does (in-window, unowned, amount <= Delta') and runs the read-explanation search;
 *     its first solution is g's choice.  After a round, g is fixed when no smaller gap that ran in the round chose one
 *     of g's transfers; a fixed gap owns its choice, and the others run again without the owned transfers.  A gap the
 *     search does not explain, or max_rounds rounds with a gap left unfixed, is cause NO_WITNESS.  D_g = the transfers
 *     g owns;
 *   - real time, one greedy pass over the reads r_1 ... r_n in the gap order, with event positions and cp = infinity
 *     for an op that never completed :ok: P_0 = -inf, P_j = max(P_{j-1}, iv(r_j), iv(t) for t in D_{j-1}); every read
 *     needs P_j < cp(r_j), every t in D_g (g >= 1) P_g < cp(t), and every :ok transfer with a window in no D_g commits
 *     after the last read and needs P_n < cp(t); otherwise cause REAL_TIME;
 *   - the counters of every gap are summed again from D_g; a mismatch is an internal error (rc < 0).
 * A VALID shard's reads and transfers are then linearizable for the per-account counters (place r_j at P_j, t in D_g
 * at max(P_g, iv(t))), and so for the bank model of ledger->bank with negative balances allowed.  Lookups are not
 * placed; `:negative-balances? false` is not decided. */
#define JTB_SW_NEVER  (-1)   /* commit_read: the transfer commits in no read's state and need not commit at all    */
#define JTB_SW_AFTER  (-2)   /* an :ok transfer that commits after every read of its shard                         */
#define JTB_SW_FREE   (-3)   /* an :ok transfer no read observes (or of amount 0): it commits inside its interval  */

typedef struct jtb_sw_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN                                                            */
    int32_t cause;              /* JTB_CAUSE_* when valid == JTB_UNKNOWN                                              */
    int32_t n_reads;            /* :ok reads of the shard                                                             */
    int32_t n_transfers;        /* transfer micro-ops of the shard (every fate)                                       */
    int64_t n_committed;        /* VALID: transfers committed in some gap                                             */
    int64_t n_committed_crashed;/* VALID: of them, the crashed ones (:info, or never completed)                       */
    int64_t n_after;            /* VALID: :ok transfers committed after the last read                                 */
    int64_t nodes;              /* search nodes of the witness rounds                                                 */
    int32_t rounds;             /* witness rounds that ran a gap of the shard                                         */
    int32_t fail_index;         /* NO_WITNESS: completion :index of the failing gap's upper read; REAL_TIME: of the read
                                   or the transfer that failed; -1                                                    */
    int64_t transfer_id;        /* REAL_TIME on a transfer: its id; -1                                                */
} jtb_sw_shard;

typedef struct jtb_sw_result {
    int32_t valid;              /* merge-valid over shards                                                            */
    int32_t n_failures;         /* shards that are not VALID                                                          */
    int64_t n_reads;
    int64_t n_transfers;
    int64_t n_committed;
    int64_t n_committed_crashed;
    int64_t n_after;
    int64_t nodes;
    int64_t rounds;             /* the most witness rounds of any shard                                               */
    double  seconds_kernel;     /* device time (CUDA events)                                                          */
    double  seconds_total;      /* host wall time of the call incl. the host pass, H2D, D2H                           */
} jtb_sw_result;

/* ---- repaired serial witness (DESIGN.md "K14 repaired serial witness") ---------------------------------------------
 * The serial-witness check, then, on a shard it leaves NO_WITNESS or REAL_TIME, up to max_repairs repair rounds.  A
 * chosen transfer is one the witness (not the transfer-placement check) put in a gap; a ban is a (gap, transfer) pair,
 * kept for good.  P^_g is the real-time point of g's lower read from the reads and the owned transfers alone.
 *   - NO_WITNESS: every gap the failing round did not explain (every unfixed gap when max_rounds ran out) steals: it
 *     gathers as a witness round does, with the chosen transfers counted as free and the repair filter below, and
 *     searches; a thief keeps its solution when no smaller thief took one of its transfers, and each chosen transfer
 *     it takes is banned in the gap that had it;
 *   - REAL_TIME: a chosen t in D_g is banned in g when cp(t) <= P_g, or when iv(t) is at or after the smallest
 *     completion of what must follow g (the reads from g's upper read on, D_h for h > g, the failing :ok transfers
 *     after the last read).
 * The gaps of the new bans and the failing gaps are released (unfixed, their choices owned by no gap), a kept thief
 * is fixed with its loot, and the witness rounds run again over the unfixed gaps; their gathers drop banned pairs and
 * every transfer with cp(t) <= P^_g.  Then the real-time pass and the re-sum run unchanged, so a VALID is the same
 * proof as the serial-witness check's.  A repair that records no new ban ends the shard's repairs.  A shard the
 * serial-witness check proves is returned as that check returns it. */
#define JTB_RW_DEFAULT_MAX_REPAIRS 32

typedef struct jtb_rw_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN                                                            */
    int32_t cause;              /* JTB_CAUSE_* when valid == JTB_UNKNOWN (of the last witness when it was repaired)   */
    int32_t n_reads;
    int32_t n_transfers;
    int64_t n_committed;        /* VALID: transfers committed in some gap                                             */
    int64_t n_committed_crashed;/* VALID: of them, the crashed ones                                                   */
    int64_t n_after;            /* VALID: :ok transfers committed after the last read                                 */
    int64_t nodes;              /* search nodes of every witness round, repairs included                              */
    int32_t rounds;             /* witness rounds that ran a gap of the shard, repairs included                       */
    int32_t fail_index;         /* as jtb_sw_shard's, of the last witness                                             */
    int64_t transfer_id;        /* as jtb_sw_shard's, of the last witness                                             */
    int32_t repairs;            /* repair rounds run on the shard                                                     */
    int32_t n_bans;             /* (transfer, gap) bans recorded                                                      */
} jtb_rw_shard;

typedef struct jtb_rw_result {
    int32_t valid;
    int32_t n_failures;
    int64_t n_reads;
    int64_t n_transfers;
    int64_t n_committed;
    int64_t n_committed_crashed;
    int64_t n_after;
    int64_t nodes;
    int64_t rounds;             /* the most witness rounds of any shard                                               */
    int64_t repairs;            /* the most repair rounds of any shard                                                */
    int64_t n_bans;
    double  seconds_kernel;
    double  seconds_total;
} jtb_rw_result;

/* ---- lifted serial witness (DESIGN.md "K15 lifted serial witness") -------------------------------------------------
 * The repaired serial witness, then, on a shard whose repairs stopped because a repair recorded no new ban (not
 * because max_repairs ran out), lift steps.  P^0_g is the real-time point of g's lower read from the reads alone.
 *   - every gap the failing round did not explain steals again as in a NO_WITNESS repair, but its gather ignores the
 *     gap's own bans (except a pair lifted before and banned again) and drops the transfers with cp(t) <= P^0_g in
 *     place of P^_g; a thief keeps its solution when no smaller thief took one of its transfers;
 *   - every ban (g, t) of a kept thief g that takes t is lifted, each chosen transfer it takes is banned in the gap
 *     that had it, and the release and the loot follow as in a repair; the repair rounds then resume unchanged.
 * A (gap, transfer) pair is lifted at most once; a lift step that lifts nothing, max_lifts lift steps, or
 * max_repairs + max_lifts repairs (lift steps included) end the shard.  The real-time pass and the re-sum run after
 * every repair, so a VALID is the serial-witness check's proof.  A shard the repaired serial witness proves, or leaves
 * after max_repairs repairs, is returned as it returns it. */
#define JTB_LW_DEFAULT_MAX_LIFTS 32

typedef struct jtb_lw_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN                                                            */
    int32_t cause;              /* JTB_CAUSE_* when valid == JTB_UNKNOWN (of the last witness)                        */
    int32_t n_reads;
    int32_t n_transfers;
    int64_t n_committed;        /* VALID: transfers committed in some gap                                             */
    int64_t n_committed_crashed;/* VALID: of them, the crashed ones                                                   */
    int64_t n_after;            /* VALID: :ok transfers committed after the last read                                 */
    int64_t nodes;              /* search nodes of every witness round, steal and lift step                           */
    int32_t rounds;             /* witness rounds that ran a gap of the shard, repairs included                       */
    int32_t fail_index;         /* as jtb_sw_shard's, of the last witness                                             */
    int64_t transfer_id;        /* as jtb_sw_shard's, of the last witness                                             */
    int32_t repairs;            /* repair rounds run on the shard, lift steps included                                */
    int32_t n_bans;             /* (gap, transfer) bans recorded, a pair banned again after its lift included        */
    int32_t lifts;              /* lift steps that lifted a ban                                                       */
    int32_t n_lifted;           /* (gap, transfer) bans lifted                                                        */
} jtb_lw_shard;

typedef struct jtb_lw_result {
    int32_t valid;
    int32_t n_failures;
    int64_t n_reads;
    int64_t n_transfers;
    int64_t n_committed;
    int64_t n_committed_crashed;
    int64_t n_after;
    int64_t nodes;
    int64_t rounds;             /* the most witness rounds of any shard                                               */
    int64_t repairs;            /* the most repair rounds of any shard                                                */
    int64_t n_bans;
    int64_t lifts;              /* the most lift steps of any shard                                                   */
    int64_t n_lifted;
    double  seconds_kernel;
    double  seconds_total;
} jtb_lw_result;

/* ---- class witness (DESIGN.md "K16 class witness") ------------------------------------------------------------------
 * The lifted serial witness, then a class pass on every shard it leaves UNKNOWN with JTB_CAUSE_UNDECIDED,
 * JTB_CAUSE_NO_WITNESS or JTB_CAUSE_REAL_TIME.  A class is the set of crashed transfers (:info, or never completed) with
 * a window that the transfer-placement check placed in no gap and that share (debit, credit, amount, M(t), A(t)); its
 * members are ordered by (invocation, id).  The class pass starts again from the transfer-placement check's owners:
 *   - the gaps with Delta' = 0 are fixed; then witness rounds (Jacobi, at most max_rounds).  Each unfixed gap gathers
 *     as a serial-witness round does, except that of each class it takes at most cap = min over the class's observed
 *     keys k of floor(Delta'_k / amount) members, the earliest unowned ones; the search keeps its chosen :ok transfers
 *     and, per class, the number x_{g,c} of members it chose;
 *   - hand-out: per class, the gaps of the round in gap order receive the unowned members at ranks
 *     [sum_{h<g} x_{h,c}, sum_{h<=g} x_{h,c}).  A gap fails when a smaller gap of the round chose one of its :ok
 *     transfers, or a member it receives does not exist or is not eligible for it (window, invocation before the upper
 *     read completes, A(t) and M(t) as in the gather).  A gap is fixed, and owns what it chose and received, when it
 *     does not fail and no gap of the round up to it that draws from one of its classes fails;
 *   - a gap with no explanation, or max_rounds with gaps left, ends the class pass (class_cause JTB_CAUSE_NO_WITNESS);
 *     otherwise the serial-witness check's real-time pass and re-sum run on the result (JTB_CAUSE_REAL_TIME when real
 *     time fails; a counter mismatch is an internal error).
 * A shard the class pass proves is VALID with the class pass's counts and commit_read; any other shard is returned as
 * the lifted serial witness returns it, with class_cause set when the class pass ran and failed. */
typedef struct jtb_cw_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN                                                            */
    int32_t cause;              /* JTB_CAUSE_* when valid == JTB_UNKNOWN (the lifted serial witness's)                */
    int32_t n_reads;
    int32_t n_transfers;
    int64_t n_committed;        /* VALID: transfers committed in some gap                                             */
    int64_t n_committed_crashed;/* VALID: of them, the crashed ones                                                   */
    int64_t n_after;            /* VALID: :ok transfers committed after the last read                                 */
    int64_t nodes;              /* search nodes of the lifted serial witness and of the class pass                    */
    int32_t rounds;             /* as jtb_lw_shard's                                                                  */
    int32_t fail_index;         /* as jtb_lw_shard's; -1 when the class pass proves the shard                         */
    int64_t transfer_id;        /* as jtb_lw_shard's; -1 when the class pass proves the shard                         */
    int32_t repairs;            /* as jtb_lw_shard's                                                                  */
    int32_t n_bans;
    int32_t lifts;
    int32_t n_lifted;
    int32_t class_cause;        /* JTB_CAUSE_NO_WITNESS / JTB_CAUSE_REAL_TIME when the class pass ran and failed, else 0 */
    int32_t class_rounds;       /* class rounds that ran a gap of the shard                                           */
    int64_t n_handed;           /* crashed transfers the class pass handed to a gap it fixed                          */
} jtb_cw_shard;

typedef struct jtb_cw_result {
    int32_t valid;
    int32_t n_failures;
    int64_t n_reads;
    int64_t n_transfers;
    int64_t n_committed;
    int64_t n_committed_crashed;
    int64_t n_after;
    int64_t nodes;
    int64_t rounds;
    int64_t repairs;
    int64_t n_bans;
    int64_t lifts;
    int64_t n_lifted;
    int64_t class_rounds;       /* the most class rounds of any shard                                                 */
    int64_t n_handed;
    double  seconds_kernel;
    double  seconds_total;
} jtb_cw_result;

/* ---- lookup witness (DESIGN.md "K17 lookup witness") ----------------------------------------------------------------
 * The class witness, then every :ok lookup of a shard it proves is placed in the shard's serial order.  A shard the
 * class witness does not prove, or with no :ok lookup, is returned as the class witness returns it.  On the others,
 * with D_g the transfers the witness commits in gap g and n the shard's reads, every transfer gets a commit gap G(t):
 * g for t in D_g; n (after the last read) for an :ok transfer in no D_g, and for a crashed transfer in no D_g that an
 * :ok lookup of the shard returns; never otherwise.  Each lookup returns exactly the transfers committed before its
 * point:
 *   - a record that names no transfer of the shard, differs from its invocation's (debit, credit, amount), names a :fail
 *     or a never-committed transfer, or repeats an id, or lo = max G over what it returns above hi = min G over the
 *     committed transfers it lacks, leaves the lookup unplaceable;
 *   - each lookup goes to the latest gap of [lo, hi] whose lower read's real-time point is below its completion; the
 *     lookups of one gap must return nested subsets of D_g, which then come in layers before each lookup;
 *   - one greedy real-time pass over the merged order of reads, transfers and lookups checks every op.
 * A failure makes the shard UNKNOWN with cause and lookup_cause JTB_CAUSE_LOOKUP, and fail_index / lookup_fail_index
 * the completion :index of the lookup that fails (for the real-time pass: the last lookup at or before the first op
 * that fails). */
typedef struct jtb_lk_shard {
    int32_t valid;              /* JTB_VALID / JTB_UNKNOWN                                                            */
    int32_t cause;              /* JTB_CAUSE_* when valid == JTB_UNKNOWN (the class witness's, or JTB_CAUSE_LOOKUP)    */
    int32_t n_reads;
    int32_t n_transfers;
    int64_t n_committed;        /* VALID: as jtb_cw_shard's                                                           */
    int64_t n_committed_crashed;
    int64_t n_after;
    int64_t nodes;
    int32_t rounds;
    int32_t fail_index;         /* as jtb_cw_shard's; the failing lookup's completion :index with JTB_CAUSE_LOOKUP    */
    int64_t transfer_id;
    int32_t repairs;
    int32_t n_bans;
    int32_t lifts;
    int32_t n_lifted;
    int32_t class_cause;
    int32_t class_rounds;
    int64_t n_handed;
    int32_t lookup_cause;       /* JTB_CAUSE_LOOKUP when the lookups of a proved shard could not be placed, else 0     */
    int32_t lookup_fail_index;  /* the completion :index of that lookup, -1 none                                      */
    int64_t n_lookups_placed;   /* VALID: :ok lookups placed in the serial order                                      */
} jtb_lk_shard;

typedef struct jtb_lk_result {
    int32_t valid;
    int32_t n_failures;
    int64_t n_reads;
    int64_t n_transfers;
    int64_t n_committed;
    int64_t n_committed_crashed;
    int64_t n_after;
    int64_t nodes;
    int64_t rounds;
    int64_t repairs;
    int64_t n_bans;
    int64_t lifts;
    int64_t n_lifted;
    int64_t class_rounds;
    int64_t n_handed;
    int64_t n_lookups_placed;
    double  seconds_kernel;
    double  seconds_total;
} jtb_lk_result;

typedef struct jtb_ctx jtb_ctx;

/* ---- lifecycle -------------------------------------------------------------------------------- */
int         jtb_abi_version(void);
/* sizeof of the ABI structs as this library was compiled, for binding self-checks:
 * 0 jtb_history, 1 jtb_model, 2 jtb_opts, 3 jtb_lin_shard, 4 jtb_lin_result, 5 jtb_setfull_shard,
 * 6 jtb_setfull_out, 7 jtb_bank_result, 8 jtb_final_config, 9 jtb_mono_shard, 10 jtb_mono_result, 11 jtb_cb_shard,
 * 12 jtb_cb_result, 13 jtb_tl_shard, 14 jtb_tl_result, 15 jtb_rx_shard, 16 jtb_rx_result, 17 jtb_rg_shard,
 * 18 jtb_rg_result, 19 jtb_tp_shard, 20 jtb_tp_result, 21 jtb_sw_shard, 22 jtb_sw_result, 23 jtb_rw_shard,
 * 24 jtb_rw_result, 25 jtb_lw_shard, 26 jtb_lw_result, 27 jtb_cw_shard, 28 jtb_cw_result, 30 jtb_lk_shard,
 * 31 jtb_lk_result, 33 jtb_edn_history, 34 jtb_edn_checks (29 and 32 are unassigned: bindings built against earlier libraries test
 * them as unknown ids); -1 otherwise */
long        jtb_struct_size(int which);
int         jtb_device_count(void);                 /* number of CUDA devices, <0 on error          */
jtb_ctx*    jtb_create(const jtb_opts* opts);       /* NULL on failure (no CUDA device etc.)        */
void        jtb_destroy(jtb_ctx* ctx);
const char* jtb_last_error(const jtb_ctx* ctx);     /* valid until the next call on ctx             */

/* ---- hot path A9: jepsen.checker/linearizable -> knossos analysis ---------------------------- *
 * Replaces (checker/linearizable {:model m}) — no call site in the reference; it would be added to
 * the compose maps at set_full.clj:156-158 / tests/ledger.clj:363-367.
 * shards[n_shards] is caller-allocated.  Returns 0 on success (verdict in out), <0 on error
 * (jtb_last_error; glue throws so that jepsen's check-safe yields {:valid? :unknown}).          */
int jtb_check_linearizable(jtb_ctx* ctx, const jtb_history* h, const jtb_model* m,
                           jtb_lin_shard* shards, jtb_lin_result* out);

/* ---- knossos analysis :configs (SURVEY §8(f) N4) ------------------------------------------------ *
 * The configurations alive where an INVALID shard got stuck: every visited configuration whose first
 * un-linearized :ok return is the witness (`:op`).  knossos reports them as {:model :pending ...} maps and
 * jepsen.checker/linearizable keeps the first 10.  Call directly after a jtb_check_linearizable(ctx, h, m, ..)
 * that reported JTB_INVALID for `shard`, with the SAME h and m (the visited table of that search is read;
 * any other call on ctx invalidates it).  Writes min(cap, *n_total) configurations in a canonical order
 * (ascending, lexicographic over the struct's int32 fields in declaration order; unused entries are 0).
 * Returns 0, <0 on error. */
typedef struct jtb_final_config {
    int32_t state;                          /* register / cas-register value (JTB_NIL = nil); 0 for bank, set */
    int32_t balances[JTB_MAX_ACCOUNTS];     /* bank: balance per account slot                                  */
    int32_t n_pending;                      /* completed ops open at the witness' return, NOT linearized
                                               (the witness itself is one of them)                             */
    int32_t n_linearized_open;              /* completed ops open at the witness' return, already linearized   */
    int32_t n_crashed_linearized;           /* crashed (:info) ops linearized in this configuration            */
    int32_t pending_index[64];              /* :index of their invocations, ascending                          */
    int32_t linearized_open_index[64];
} jtb_final_config;
int jtb_final_configs(jtb_ctx* ctx, const jtb_history* h, const jtb_model* m, int32_t shard,
                      jtb_final_config* out, int32_t cap, int64_t* n_total);

/* ---- hot path A4: (checker/set-full {:linearizable? L}) at set_full.clj:157 ------------------ */
int jtb_check_set_full(jtb_ctx* ctx, const jtb_history* h, int linearizable, jtb_setfull_out* out);

/* ---- hot path A8: bank SI checker, tests/ledger.clj:154-192 (after ledger->bank) -------------- *
 * accounts->n_accounts must lie in [0, JTB_MAX_ACCOUNTS] (0: every key a read shows is :unexpected-key); <0 otherwise,
 * with jtb_last_error saying why (the context stays usable). */
int jtb_check_bank_totals(jtb_ctx* ctx, const jtb_history* h, const jtb_model* accounts,
                          int64_t total_amount, jtb_bank_result* out);

/* ---- monotonic-key check (see jtb_mono_shard above) ------------------------------------------------------------ *
 * shards[n_shards] is caller-allocated.  Returns 0 on success, <0 on a malformed read payload (length not a multiple
 * of 3, out of range, a key twice in one read), more than 2^31-1 reads, or when the device cannot hold the dense
 * value matrix (jtb_last_error says which). */
int jtb_check_monotonic_keys(jtb_ctx* ctx, const jtb_history* h, int32_t flags, jtb_mono_shard* shards,
                             jtb_mono_result* out);

/* ---- counter-bounds check (see jtb_cb_shard above) -------------------------------------------------------------- *
 * shards[n_shards] is caller-allocated; flags is reserved and must be 0.  Returns 0 on success, <0 on a malformed read
 * payload (as jtb_check_monotonic_keys), a transfer with a negative amount or an account outside [0, 2^30), more than
 * 2^31-1 reads or (transfer, observed key) contributions, flags != 0, or a device allocation failure (jtb_last_error
 * says which; the context stays usable). */
int jtb_check_counter_bounds(jtb_ctx* ctx, const jtb_history* h, int32_t flags, jtb_cb_shard* shards,
                             jtb_cb_result* out);

/* ---- transfer-lookup check (see jtb_tl_shard above) ------------------------------------------------------------- *
 * shards[n_shards] is caller-allocated; flags is reserved and must be 0.  Returns 0 on success, <0 on a malformed read
 * payload (as jtb_check_monotonic_keys), a transfer or lookup payload whose length is not a multiple of 5, a transfer
 * invoke without ids, two transfer invokes of one shard carrying the same id, a negative amount or an account outside
 * [0, 2^30) in a transfer invoke, more than 2^31-1 records or reads, an S matrix (lookups x observed keys) the device
 * cannot hold, flags != 0, or a device allocation failure (jtb_last_error says which; the context stays usable). */
int jtb_check_transfer_lookups(jtb_ctx* ctx, const jtb_history* h, int32_t flags, jtb_tl_shard* shards,
                               jtb_tl_result* out);

/* ---- read-explanation check (see jtb_rx_shard above) ------------------------------------------------------------ *
 * shards[n_shards] is caller-allocated; max_nodes <= 0 means JTB_RX_DEFAULT_MAX_NODES; flags is reserved and must be 0.
 * Returns 0 on success, <0 on the transfer-lookup check's input errors, flags != 0, or a device allocation failure
 * (jtb_last_error says which; the context stays usable). */
int jtb_check_read_explanations(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t flags,
                                jtb_rx_shard* shards, jtb_rx_result* out);

/* ---- read-gap check (see jtb_rg_shard above) -------------------------------------------------------------------- *
 * shards[n_shards] is caller-allocated; max_nodes <= 0 means JTB_RG_DEFAULT_MAX_NODES; flags is reserved and must be 0.
 * Returns 0 on success, <0 on the read-explanation check's input errors, flags != 0, a dense value matrix (reads x
 * keys of the full-key shards) the device cannot hold, or a device allocation failure (jtb_last_error says which; the
 * context stays usable). */
int jtb_check_read_gaps(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t flags, jtb_rg_shard* shards,
                        jtb_rg_result* out);

/* ---- transfer-placement check (see jtb_tp_shard above) -------------------------------------------------------- *
 * shards[n_shards] is caller-allocated; max_nodes <= 0 means JTB_TP_DEFAULT_MAX_NODES, max_rounds <= 0
 * JTB_TP_DEFAULT_MAX_ROUNDS; flags is reserved and must be 0.  Returns 0 on success, <0 on the read-gap check's errors
 * (jtb_last_error says which; the context stays usable). */
int jtb_check_transfer_placement(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                                 int32_t flags, jtb_tp_shard* shards, jtb_tp_result* out);

/* ---- serial-witness check (see jtb_sw_shard above) ------------------------------------------------------------ *
 * shards[n_shards] is caller-allocated; max_nodes and max_rounds as for jtb_check_transfer_placement (and passed to
 * it); flags is reserved and must be 0.  commit_read may be NULL, else it receives one entry per transfer micro-op in
 * history order: the completion :index of the first read whose state holds the transfer, JTB_SW_NEVER, JTB_SW_AFTER or
 * JTB_SW_FREE (JTB_SW_NEVER for every transfer of a shard that is not VALID).  Returns 0 on success, <0 on the
 * transfer-placement check's errors or when the counters of a witness do not add up (jtb_last_error says which; the
 * context stays usable). */
int jtb_check_serial_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t flags,
                             int32_t* commit_read, jtb_sw_shard* shards, jtb_sw_result* out);

/* ---- repaired serial witness (see jtb_rw_shard above) ---------------------------------------------------------- *
 * As jtb_check_serial_witness; max_rounds bounds each run of the witness rounds (the first and one per repair);
 * max_repairs <= 0 means JTB_RW_DEFAULT_MAX_REPAIRS; flags is reserved and must be 0. */
int jtb_check_repaired_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                               int32_t max_repairs, int32_t flags, int32_t* commit_read, jtb_rw_shard* shards,
                               jtb_rw_result* out);

/* ---- lifted serial witness (see jtb_lw_shard above) ------------------------------------------------------------ *
 * As jtb_check_repaired_witness; max_lifts <= 0 means JTB_LW_DEFAULT_MAX_LIFTS; flags is reserved and must be 0. */
int jtb_check_lifted_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                             int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t* commit_read,
                             jtb_lw_shard* shards, jtb_lw_result* out);

/* ---- class witness (see jtb_cw_shard above) -------------------------------------------------------------------- *
 * As jtb_check_lifted_witness, with the same budgets; max_rounds also bounds the class rounds; flags is reserved and
 * must be 0. */
int jtb_check_class_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                            int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t* commit_read,
                            jtb_cw_shard* shards, jtb_cw_result* out);

/* ---- lookup witness (see jtb_lk_shard above) ------------------------------------------------------------------- *
 * As jtb_check_class_witness, with the same budgets; flags is reserved and must be 0.  commit_read (may be NULL) as
 * the class witness's, except that a crashed transfer committed after the last read because a lookup returns it is
 * JTB_SW_AFTER.  lookup_read (may be NULL) gets one entry per :ok lookup in history order: the completion :index of
 * the read the lookup precedes in the serial order, JTB_SW_AFTER after the last read, and JTB_SW_NEVER for every lookup
 * of a shard that is not VALID. */
int jtb_check_lookup_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                             int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t* commit_read,
                             int32_t* lookup_read, jtb_lk_shard* shards, jtb_lk_result* out);

/* ---- K18: a stored ledger history.edn read on the device ------------------------------------------------------ *
 * The bytes of a Jepsen history.edn (one op map per top-level form, optionally tagged #jepsen.history.Op{...}, or one
 * top-level vector of op maps) flattened into one of the ledger forms: exactly the arrays of the Python path
 * edn.read_history + history.flatten_ops(ops, form), and meta["multi_transfer_txns"] (0 for JTB_FORM_BANK).  The
 * history is one shard (key id -1).  Its arrays are page-locked host memory the library owns (jtb_host_alloc); release
 * them with jtb_edn_history_free.  The EDN read is the subset Jepsen's store writes: keys in any order, unknown keys
 * with arbitrary values, integers with an optional N suffix, nil, true, false, keywords, strings with escapes and ','
 * as whitespace; ';' comments, #_ discard, character literals and a float where an integer is read are refused.
 * Returns 0, or <0 where the Python path raises or the EDN is unsupported, with jtb_last_error giving the byte and the
 * reason (out is left empty; the context stays usable).  flags is reserved and must be 0. */
#define JTB_FORM_BANK            0   /* flatten_ops(..., "bank")            */
#define JTB_FORM_LEDGER_COUNTERS 1   /* flatten_ops(..., "ledger-counters") */
#define JTB_FORM_LEDGER_LOOKUPS  2   /* flatten_ops(..., "ledger-lookups")  */
typedef struct jtb_edn_history {
    jtb_history history;
    int64_t multi_transfer_txns;   /* transfer invokes with more than one micro-op (ledger forms)          */
    int64_t n_ops;                 /* top-level op maps read, client and nemesis alike                      */
    double  seconds_h2d;           /* copy of the text to the device                                        */
    double  seconds_kernel;        /* device passes (CUDA events)                                           */
    double  seconds_d2h;           /* copy of the arrays back into page-locked host memory                  */
    double  seconds_total;
} jtb_edn_history;
int  jtb_read_ledger_edn(jtb_ctx* ctx, const char* text, int64_t n_bytes, int32_t form, int32_t flags,
                         jtb_edn_history* out);
void jtb_edn_history_free(jtb_edn_history* out);

/* ---- K19: the host checks of a ledger compose on a stored history.edn ------------------------------------------ *
 * The bytes jtb_read_ledger_edn reads, summarised for the checkers unexpected-ops, lookup-all-invoked-transfers,
 * final-reads and stats (tests/ledger.clj:194-282, jepsen.checker/stats) as they run on the op maps of
 * edn.read_history: a missing :index or :time counts as 0, and a txn's tag is its first micro-op's (an empty value has
 * none).  Client ops are those with an integer :process.  Reported per flagged op: its ordinal among the top-level op
 * maps, the bytes of its map, its :index and :time with their presence, and where they apply its class of equal
 * :value and its suspect bit.  The flagged ops' arrays are page-locked host memory the library owns; release them with
 * jtb_edn_checks_free.  Where the summary could differ from those checkers the call refuses the input instead:
 * refused = 1, refused_at = the byte (-1 none) and refused_reason; the arrays are then empty.  It refuses whatever
 * jtb_read_ledger_edn refuses in JTB_FORM_LEDGER_LOOKUPS; a micro-op of a :final? :ok read or lookup that is not
 * [keyword id map-or-nil] with an int64 id; a key of its map other than :debit-acct :credit-acct :amount
 * :debits-posted :credits-posted, or a value there that is not an int64 or nil; a transfer invoke's id that is not an
 * int64; and a collision of the 128-bit digests that group equal final values.  Returns 0 (refused or not), <0 on
 * malformed arguments, CUDA and allocation errors.  flags is reserved and must be 0. */
typedef struct jtb_edn_flag {
    int64_t op;          /* ordinal among the top-level op maps                                                  */
    int64_t begin, end;  /* the op map's bytes [begin, end), from its '{' (a tag before it is not included)       */
    int64_t time;        /* :time, 0 when absent                                                                  */
    int64_t first;       /* open invokes: the ordinal of the first invoke of the process's last run of invokes
                            (where unexpected-ops puts the process in its map); -1 otherwise                      */
    int32_t index;       /* :index, 0 when absent                                                                 */
    int32_t cls;         /* final reads and final lookups: the class of equal :value, from 0 per kind; -1 otherwise */
    uint8_t has_time, has_index;
    uint8_t suspect;     /* final lookups: the lookup lacks an id some transfer invoke has                         */
    uint8_t pad[5];
} jtb_edn_flag;
typedef struct jtb_edn_checks {
    int64_t n_ops;             /* top-level op maps read, client and nemesis alike                                  */
    int64_t n_client;          /* ops with an integer :process                                                      */
    int64_t n_ok, n_fail, n_info;   /* client completions by :type (every client op is :f :txn)                    */
    int64_t n_open;            /* invokes that are the last client op of their process                             */
    int64_t n_final_reads, n_final_lookups;   /* :final? :ok ops whose first micro-op is :r, :l-t              */
    int64_t n_read_classes, n_lookup_classes; /* distinct :value among them                                       */
    int64_t n_invoked;         /* distinct ids of the micro-ops of :t invokes                                       */
    int64_t n_suspect;         /* final lookups that lack one of them                                               */
    jtb_edn_flag last;         /* the last client op (op = -1: none)                                                */
    jtb_edn_flag* open;        /* n_open, by :process                                                              */
    jtb_edn_flag* fails;       /* n_fail, in history order                                                          */
    jtb_edn_flag* final_reads; /* n_final_reads, in history order                                                   */
    jtb_edn_flag* final_lookups;   /* n_final_lookups, in history order                                             */
    int32_t refused, reserved;
    int64_t refused_at;
    char    refused_reason[128];
    double  seconds_h2d;       /* copy of the text to the device                                                    */
    double  seconds_kernel;    /* device passes (CUDA events)                                                       */
    double  seconds_d2h;       /* copy of the flagged ops back                                                      */
    double  seconds_total;
} jtb_edn_checks;
int  jtb_ledger_edn_checks(jtb_ctx* ctx, const char* text, int64_t n_bytes, int32_t flags, jtb_edn_checks* out);
void jtb_edn_checks_free(jtb_edn_checks* out);

/* ---- K20: a stored set-full history.edn read on the device ----------------------------------------------------- *
 * The bytes of a set-full history.edn (set_full.clj:29-45, 107-134; the EDN subset and op fields of K18) flattened into
 * the keyed set form: exactly the arrays of edn.read_history(text, independent=True) + history.flatten_ops(ops, "set").
 * A 2-element vector or list :value is a jepsen.independent tuple [key value]; each integer key is one shard, in
 * ascending key order, and the events whose key is nil or whose :value is not a tuple form the last shard, key id -1
 * (even when a real key -1 exists).  An :add of a nil value is dropped; a :read of nil has payload_len -1, of a set
 * literal its members sorted ascending, of a vector or list its members in order.  multi_transfer_txns is 0.  Refused
 * (rc < 0, jtb_last_error naming the first offending byte): whatever K18 refuses about the EDN and the op fields, :f
 * other than :add or :read on a client op, a key that is not an integer or nil or lies outside int64, an add value or
 * member that is not an integer or lies outside int32, a read value that is not nil or a collection, a set literal with
 * a repeated member, and more than 2^31 - 3 members.  Release the arrays with jtb_edn_history_free.  flags is reserved
 * and must be 0. */
int  jtb_read_set_edn(jtb_ctx* ctx, const char* text, int64_t n_bytes, int32_t flags, jtb_edn_history* out);

/* ---- multi-GPU fan-out inside the library (SURVEY §8(b) `n_gpus`, §8(e)) ----------------------------------- *
 * What `independent/checker` (set_full.clj:155) does over JVM threads, done over the GPUs of one box for a host
 * that is a single process (a JVM through JNI): the shards (independent keys) of the history are partitioned over
 * `n_gpus` devices (longest-processing-time-first on events^2), every device checks its share through its own
 * context on its own host thread, and the per-shard (verdict, witness, previous-ok) vectors are merged with ONE
 * ncclAllReduce(ncclMax) over int32[3 * n_shards] (ncclCommInitAll inside the library; NCCL is dlopen'ed at
 * jtb_multi_create, libjtb_check.so itself has no link-time dependency on it).  No configuration ever crosses GPUs:
 * linearizability is local (Herlihy-Wing), so the verdict lattice 0 < 1 < 2 under MAX is all that has to travel.
 * A history with ONE shard runs on the first device (it does not shard: SURVEY §8(e) "replicas only").
 * opts->device is ignored (devices 0 .. n_gpus-1); n_gpus <= 0 means every visible device.                     */
typedef struct jtb_multi jtb_multi;
jtb_multi*  jtb_multi_create(const jtb_opts* opts, int n_gpus);   /* NULL on failure (see jtb_multi_create_error) */
const char* jtb_multi_create_error(void);                          /* why the last jtb_multi_create returned NULL   */
void        jtb_multi_destroy(jtb_multi* mg);
int         jtb_multi_n_gpus(const jtb_multi* mg);
const char* jtb_multi_last_error(const jtb_multi* mg);
/* same contract as jtb_check_linearizable; out->seconds_kernel = max over devices; device_of_shard (may be NULL)
 * receives the device each shard was checked on */
int jtb_multi_check_linearizable(jtb_multi* mg, const jtb_history* h, const jtb_model* m,
                                 jtb_lin_shard* shards, jtb_lin_result* out, int32_t* device_of_shard);
/* same contract as jtb_check_set_full; only the per-shard structs are merged (the optional per-element and
 * suspect-read detail of `out` must be unset: elem_capacity == suspect_capacity == missing_capacity == 0) */
int jtb_multi_check_set_full(jtb_multi* mg, const jtb_history* h, int linearizable, jtb_setfull_out* out,
                             int32_t* device_of_shard);

/* ---- diagnostics: counters of the last jtb_check_linearizable call ------------------------------ *
 * out[0..11] = configs, probes, expansions, ring tail, ring head, idle polls, max probe length,
 * table slots, grid CTAs, ring entries, search launches (pause/resume growth + 1), kernel microseconds,
 * out[12..14] = host->device bytes, device->host bytes, CUDA kernels launched,
 * out[15..18] = scout steps, scout configs, shards decided by a scout, scouts launched */
int jtb_get_stats(jtb_ctx* ctx, unsigned long long* out, int n);

/* SURVEY 8(f) N2 — the step before the checkers, on the device.
 * jtb_partition_by_key replaces jepsen.independent/subhistory (set_full.clj:155: independent/checker re-filters the
 * whole history once per key): ONE stable partition of the events by key.  event_key[i] = the key of event i (any
 * int64; nemesis / un-keyed events can carry a key of their own).  Out: order[n_events] = original position of the
 * i-th event of the partitioned history (events of one key keep their history order), key_ids[n_keys] ascending,
 * shard_off[n_keys + 1] = the CSR offsets of jtb_history; key_cap = capacity of key_ids (shard_off: key_cap + 1).
 * Returns <0 with "key_cap too small" when the history has more than key_cap keys (order is written, shard_off and
 * key_ids are not, *n_keys = 0; the context stays usable).
 * jtb_ledger_balances is ledger->bank's arithmetic (tests/ledger.clj:100-105): balance = credits-posted - debits-posted,
 * computed in int64 and truncated to its low 32 bits (two's complement) when the difference leaves int32. */
int jtb_partition_by_key(jtb_ctx* ctx, int64_t n_events, const int64_t* event_key, int32_t* order, int64_t* shard_off,
                         int64_t* key_ids, int32_t key_cap, int32_t* n_keys);
int jtb_ledger_balances(jtb_ctx* ctx, int64_t n, const int64_t* credits_posted, const int64_t* debits_posted,
                        int32_t* balance);

/* Page-locked host memory for the flattened arrays (what a JNI shim wraps in a direct ByteBuffer, what the Python
 * mirror backs its numpy arrays with).  Not required: any host pointer works; page-locked ones are copied by DMA at the
 * PCIe rate instead of being staged through the driver (the id lists of 100k-op set-full histories are ~600 MB).
 * NULL when the allocation fails. */
void* jtb_host_alloc(size_t bytes);
void  jtb_host_free(void* p);

/* ---- diagnostics: host preparation only (pairing, slots, tables) — no device work; returns seconds
 * or a negative value on malformed input.  Lets callers see the host share of time-to-verdict. */
double jtb_prepare_seconds(const jtb_history* h, const jtb_model* m);
/* same, also reporting the layout chosen: info[0..3] = key bytes, slot lanes (32|64), max crashed-op classes per
 * shard, total completed ops (ranks) */
double jtb_prepare_info(const jtb_history* h, const jtb_model* m, long long info[4]);

/* ---- K2 in isolation: visited-table probe/insert microbenchmark (roofline evidence) ----------- *
 * Inserts n_keys pseudo-random 128-bit keys then probes them `rounds` times; returns device
 * seconds for insert and probe phases.  variant selects the probe path (see DESIGN.md).          */
int jtb_table_bench(jtb_ctx* ctx, uint64_t n_keys, int variant, int rounds,
                    double* insert_seconds, double* probe_seconds, uint64_t* found);

/* ---- the memory system under a hash probe: random 16 B gathers as a function of the footprint ------------------ *
 * Every thread issues `iters` rounds of `in_flight` (1, 2, 4, 8, 16) independent random 16 B loads (the search
 * kernel's ld.global.cg.v2.u64 probe; wide = 2: both halves of the 32 B sector) over a table of table_bytes
 * (rounded down to a power of two), ctas_per_sm x 256 threads per SM.  Returns the best of `rounds` timings and the
 * number of 16 B-slot probes issued.  scripts/probe_sweep.py runs it over table sizes and in-flight depths.     */
int jtb_gather_bench(jtb_ctx* ctx, uint64_t table_bytes, int in_flight, int wide, uint32_t iters, int ctas_per_sm,
                     int rounds, double* seconds, uint64_t* n_probes);

#ifdef __cplusplus
}
#endif
#endif /* JTB_CHECK_H */
