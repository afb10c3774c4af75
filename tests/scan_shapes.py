"""History builders at the shapes where the scan kernels switch code path (plain Python, no device).

set-full (`jtb_check_set_full`, csrc/jtb_scans.cuh): the 32-bit words of the read x element bit matrix, the 128-word
tiles and 512-read chunks of the column scan (partial results merge through 64-bit atomics), the `n_elig` eligibility
prefix, the direct versus sorted id table, duplicates, final reads, the millisecond latency boundary, degenerate shards
and more shards than one grid dimension holds.  bank totals (`jtb_check_bank_totals`): every outcome type, the rule
precedence, ties, float-rounded badness, int32 extremes and multi-block atomics.  partition (`jtb_partition_by_key`,
`jtb_ledger_balances`): block edges, the sign flip of the radix key, int32 truncation.

Every builder returns a FlatHistory (numpy arrays for the partition); sf_id_tables' `meta["lookup"]` names the id
table each of its shards takes.
"""
from __future__ import annotations

import numpy as np

from jepsen_tigerbeetle_b200 import history as H

INT32_MIN, INT32_MAX = -(2 ** 31), 2 ** 31 - 1
INT64_MIN, INT64_MAX = -(2 ** 63), 2 ** 63 - 1
RCHUNK = 512          # reads per chunk of the set-full column scan
GRID_YZ_MAX = 65535   # CUDA's cap on gridDim.y and gridDim.z
ACCOUNTS = tuple(range(1, 9))


class Script:
    """A Jepsen history written op by op: :index = position, :time in ns (one millisecond per op unless given)."""

    def __init__(self, key=None):
        self.ops: list[dict] = []
        self.key = key
        self.t = 0

    def op(self, p, type_, f, value=None, time=None, final=False):
        self.t = self.t + 1_000_000 if time is None else int(time)
        o = {"process": p, "type": type_, "f": f, "value": value if self.key is None else (self.key, value),
             "index": len(self.ops), "time": self.t}
        if final:
            o["final?"] = True
        self.ops.append(o)
        return self

    def add(self, p, v, outcome="ok"):
        """:add v invoked by p and completed with `outcome` (None: never completes)."""
        self.op(p, "invoke", "add", v)
        if outcome:
            self.op(p, outcome, "add", v)
        return self

    def read(self, p, value, outcome="ok", final=False):
        """A read by p returning `value` (a list keeps its order and repeats) when `outcome` is :ok."""
        self.op(p, "invoke", "read", None, final=final)
        if outcome:
            self.op(p, outcome, "read", value if outcome == "ok" else None, final=final)
        return self

    def flat(self, model="set") -> H.FlatHistory:
        return H.flatten_ops(self.ops, model)


def lookup_path(ids) -> str:
    """Which id -> position table run_set_full builds for a shard tracking `ids`: a direct table when the span is at
    most 4n + 1024, a sorted (id, position) table otherwise."""
    ids = sorted(set(int(x) for x in ids))
    if not ids:
        return "none"
    return "direct" if ids[-1] - ids[0] + 1 <= 4 * len(ids) + 1024 else "sorted"


def tracked_ids(h: H.FlatHistory, s: int) -> list[int]:
    """The values :add-invoked in shard s (the elements set-full tracks there)."""
    lo, hi = int(h.shard_off[s]), int(h.shard_off[s + 1])
    sel = (h.process[lo:hi] >= 0) & (h.f[lo:hi] == H.F_ADD) & (h.type[lo:hi] == H.T_INVOKE)
    return sorted(set(h.a[lo:hi][sel].tolist()))


def keys(parts, meta=None) -> H.FlatHistory:
    h = H.concat_keys(parts)
    h.meta = dict(meta or {})
    return h


# =====================================================================================================================
# set-full
# =====================================================================================================================
def sf_elements(n: int, seed: int = 0) -> H.FlatHistory:
    """One shard tracking n elements (ids 3n-1 .. 2n, so positions and ids run in opposite orders), then four reads
    whose membership patterns change across every word (and, for n >= 4096, tile) edge.  The last read is final and
    misses the last element only, so its suspect row ends in a partial word."""
    rng = np.random.default_rng(seed)
    ids = [3 * n - 1 - i for i in range(n)]
    s = Script()
    for i, v in enumerate(ids):
        s.add(0, v, "ok" if i % 7 else "info")
    pos = np.arange(n)
    for mask in (pos % 3 != 0, pos % 2 == 0, rng.random(n) < 0.8):
        s.read(1, [v for v, m in zip(ids, mask) if m])
    s.read(1, ids[:-1], final=True)
    return s.flat()


def sf_reads(n_reads: int, n_elems: int = 70, seed: int = 0) -> H.FlatHistory:
    """One shard read n_reads times.  Every fourth pair of reads overlaps with its completions swapped, so completion
    order differs from invocation order.  The deciding reads of a few elements sit in different 512-read chunks:
      e0 present only in read 0;                e1 present only in the last read;
      e2 present in chunk 0, absent from chunk 1 on;   e3 absent until chunk 2 (or the last read), present after;
      e4 :info add first seen by the last read (it fixes `known` in the last chunk);
      e5 :info add present from the middle read on;   e6 absent only in the middle read;
      e7 present only in read 511, e8 only in read 512;
    the rest random (97 % present).  Elements n_elems-5 .. n_elems-1 are invoked just before read k and complete after
    it (k = n_reads // 3 + j), so n_elig changes inside a chunk."""
    rng = np.random.default_rng(seed)
    R, late = n_reads, list(range(n_elems - 5, n_elems))
    late_at = {R // 3 + j: e for j, e in enumerate(late)}
    s = Script()
    for e in range(n_elems - 5):
        s.add(0, e, "info" if e in (4, 5) else "ok")
    ks = np.arange(R)
    M = rng.random((R, n_elems)) < 0.97      # M[k, e]: read k shows element e
    for e, col in enumerate((ks == 0, ks == R - 1, ks < RCHUNK, ks >= min(2 * RCHUNK, R - 1), ks == R - 1,
                             ks >= R // 2, ks != R // 2, ks == RCHUNK - 1, ks == RCHUNK)):
        M[:, e] = col
    for q, e in late_at.items():
        M[:q + 1, e] = False

    def value(k):
        return np.flatnonzero(M[k]).tolist()

    k = 0
    while k < R:
        k0 = k
        if k0 in late_at:
            s.op(0, "invoke", "add", late_at[k0])
        if k0 % 8 == 0 and k0 + 1 < R and k0 + 1 not in late_at:
            s.op(1, "invoke", "read").op(2, "invoke", "read")
            s.op(2, "ok", "read", value(k0 + 1)).op(1, "ok", "read", value(k0))
            k += 2
        else:
            s.read(1, value(k0))
            k += 1
        if k0 in late_at:
            s.op(0, "ok", "add", late_at[k0])
    return s.flat()


ELIG_TARGETS = (0, 1, 31, 32, 33, 63, 64, 65)


def sf_elig(seed: int = 0) -> H.FlatHistory:
    """Reads that complete after exactly n_elig add invokes for n_elig in ELIG_TARGETS, each holding ids added before it
    and ids whose add has not been invoked yet (their bits are set but lie past the eligibility prefix).  One read is
    invoked before the 30th add and completes after the 66th."""
    rng = np.random.default_rng(seed)
    n = 70
    s = Script()
    s.op(2, "invoke", "read")
    for i in range(n + 1):
        if i in ELIG_TARGETS:
            seen = [v for v in range(i) if rng.random() < 0.7]
            s.read(1, sorted(seen + [i, i + 1, n + 5]))
        if i == 30:
            s.op(3, "invoke", "read")
        if i == 66:
            s.op(3, "ok", "read", list(range(0, 66, 2)))
        if i < n:
            s.add(0, i)
    s.op(2, "ok", "read", list(range(1, n, 3)))
    s.read(1, list(range(n)))
    return s.flat()


def _id_table_key(ids, extra_reads=()) -> H.FlatHistory:
    s = Script()
    for v in ids:
        s.add(0, v)
    s.read(1, sorted(ids))
    s.read(1, sorted(ids)[1::2])
    lo, hi = min(ids), max(ids)
    untracked = [x for x in (lo - 1, hi + 1, lo + 1 if lo + 1 not in ids else None) if x is not None
                 and INT32_MIN <= x <= INT32_MAX]
    s.read(1, sorted(set(ids[::3]) | set(untracked)))
    for r in extra_reads:
        s.read(1, r)
    return s.flat()


def sf_id_tables() -> H.FlatHistory:
    """Five keys, each tracking 8 or 9 ids: span exactly 4n + 1024 (direct table), 4n + 1025 (sorted), negative ids on
    a direct table, sparse negative ids (sorted), and INT32_MIN, -1, 0, 1, INT32_MAX (sorted).  Reads also hold
    untracked ids just outside and inside each table.  meta["lookup"] is the path each shard takes."""
    n = 8
    direct = [100 + i for i in range(n - 1)] + [100 + 4 * n + 1023]
    sorted_ = [100 + i for i in range(n - 1)] + [100 + 4 * n + 1024]
    neg = [-5000 + 7 * i for i in range(n)]
    neg_sparse = [-(10 ** 6) * (i + 1) for i in range(n)]
    extremes = [INT32_MIN, -1, 0, 1, INT32_MAX]
    parts = [_id_table_key(direct), _id_table_key(sorted_), _id_table_key(neg),
             _id_table_key(neg_sparse), _id_table_key(extremes, extra_reads=[[INT32_MIN, 0, INT32_MAX]])]
    return keys(parts, {"lookup": ["direct", "sorted", "direct", "sorted", "sorted"]})


def sf_add_free_duplicate() -> H.FlatHistory:
    """No :add at all; one read repeats an id: jepsen's (frequencies v) counts it, so duplicated_count = 1 and the key
    is :invalid."""
    return Script().read(0, [7, 7]).flat()


def sf_duplicates() -> H.FlatHistory:
    """Keys: tracked ids repeated at bits 0 and 31 of word 0 and bits 0 and 31 of word 1 (multiplicities 2, 3, 2, 4);
    an untracked id repeated next to a tracked one; an id repeated in a read before its add is invoked; an add-free key
    whose read repeats an id (the bug-1 shape as one key among keys with adds); an add-free key without repeats."""
    a = Script()
    for v in range(64):
        a.add(0, v)
    a.read(1, list(range(64)) + [0, 31, 31, 32, 63, 63, 63])
    b = Script().add(0, 1).read(1, [1, 7, 7])
    c = Script().read(1, [5, 5, 6]).add(0, 5).read(1, [5])
    d = Script().read(0, [7, 9, 7])
    e = Script().read(0, [3, 4], final=True)
    return keys([x.flat() for x in (a, b, c, d, e)])


def sf_readd() -> H.FlatHistory:
    """Re-added elements: 1 is re-added with reads between the two invokes and between the second invoke and its :ok;
    2's second add crashes (:info); 3 is re-added after being lost."""
    s = Script()
    s.add(0, 1).add(0, 2).add(0, 3)
    s.read(1, [1, 2, 3]).read(1, [2])
    s.op(0, "invoke", "add", 1)
    s.read(1, [2]).read(1, [1, 2])
    s.op(0, "ok", "add", 1)
    s.add(0, 2, "info").read(1, [1])
    s.add(0, 3).read(1, [1, 3]).read(1, [1, 2, 3])
    return s.flat()


def sf_read_outcomes() -> H.FlatHistory:
    """:fail, :info and never-completed reads between :ok ones: only :ok reads constrain the elements."""
    s = Script()
    s.add(0, 1).add(0, 2)
    s.read(1, None, outcome="fail")
    s.read(2, None, outcome="info")
    s.read(3, None, outcome=None)
    s.read(4, [1]).read(4, [1, 2])
    s.read(5, None, outcome="fail").read(5, [2])
    s.add(0, 3, outcome=None)
    s.read(6, [1, 2, 3], outcome="info")
    return s.flat()


def sf_finals() -> H.FlatHistory:
    """Final reads: one misses the elements at positions 31 and 32 (ids 1000 - position); a key with no elements has a
    final read; a key has two final reads missing different elements; a crashed final read is ignored."""
    a = Script()
    for i in range(40):
        a.add(0, 1000 - i)
    a.read(1, [1000 - i for i in range(40) if i not in (31, 32)], final=True)
    b = Script().read(1, [], final=True).read(1, [4, 5], final=True)
    c = Script()
    for v in range(10):
        c.add(0, v)
    c.read(1, list(range(1, 10)), final=True).read(2, list(range(9)), final=True)
    c.read(3, None, outcome="info", final=True)
    return keys([a.flat(), b.flat(), c.flat()])


LATENCY_GAPS_NS = (999_999, 1_000_000, 1_000_001)


def sf_latency() -> H.FlatHistory:
    """Three keys, one element each: added (:ok at K = 10 ms), absent from a read invoked at K + d - 1, present in the
    next; d = stable_time - known_time runs over LATENCY_GAPS_NS, so the stable latency is 0, 1 and 1 ms and the last
    two keys are stale (:invalid under {:linearizable? true})."""
    parts = []
    K = 10_000_000
    for d in LATENCY_GAPS_NS:
        s = Script()
        s.op(0, "invoke", "add", 1, time=0).op(0, "ok", "add", 1, time=K)
        s.op(1, "invoke", "read", time=K + d - 1).op(1, "ok", "read", [], time=K + d)
        s.op(1, "invoke", "read", time=K + d + 1).op(1, "ok", "read", [1], time=K + d + 2)
        parts.append(s.flat())
    return keys(parts)


def sf_degenerate() -> H.FlatHistory:
    """Keys with no events, reads only, adds only, nemesis events only (process < 0), and one ordinary key."""
    empty = Script().flat()
    reads_only = Script().read(0, [1, 2]).read(0, [], final=True).flat()
    adds_only = Script().add(0, 1).add(0, 2, "info").add(0, 3, None).flat()
    nemesis = Script().add(0, 1).read(1, [1, 1]).flat()
    nemesis.process[:] = -1
    normal = Script().add(0, 1).add(0, 2).read(1, [1, 2]).read(1, [2]).flat()
    return keys([empty, reads_only, adds_only, nemesis, normal])


def sf_many_keys(n_keys: int = 70_000) -> H.FlatHistory:
    """n_keys keys (more than the 65,535 one grid dimension holds), each one add and one read: the read shows the
    element (stable), misses it (k % 7 == 3: lost) or repeats it (k % 11 == 5: duplicated)."""
    ops = []
    for k in range(n_keys):
        v = [] if k % 7 == 3 else [k, k] if k % 11 == 5 else [k]
        for o in ({"process": 0, "type": "invoke", "f": "add", "value": (k, k)},
                  {"process": 0, "type": "ok", "f": "add", "value": (k, k)},
                  {"process": 1, "type": "invoke", "f": "read", "value": (k, None)},
                  {"process": 1, "type": "ok", "f": "read", "value": (k, v)}):
            o["index"] = len(ops)
            o["time"] = len(ops) * 1000
            ops.append(o)
    return H.flatten_ops(ops, "set")


ELEMENT_COUNTS = (1, 31, 32, 33, 63, 64, 65, 4095, 4096, 4097)
READ_COUNTS = (511, 512, 513, 1025)

# name -> builder of every set-full shape (the many-key one aside: it is large enough to get tests of its own)
SF_SHAPES = {
    **{f"elements-{n}": (lambda n=n: sf_elements(n)) for n in ELEMENT_COUNTS},
    **{f"reads-{r}": (lambda r=r: sf_reads(r)) for r in READ_COUNTS},
    "reads-1025-elements-4097": lambda: sf_reads(1025, 4097, seed=1),
    "elig": sf_elig, "id-tables": sf_id_tables, "add-free-duplicate": sf_add_free_duplicate,
    "duplicates": sf_duplicates, "re-add": sf_readd, "read-outcomes": sf_read_outcomes, "finals": sf_finals,
    "latency": sf_latency, "degenerate": sf_degenerate, "empty": lambda: Script().flat(),
}


# =====================================================================================================================
# bank totals
# =====================================================================================================================
ZERO = {a: 0 for a in ACCOUNTS}


def _bank(reads, transfers=0) -> H.FlatHistory:
    s = Script()
    for i in range(transfers):
        s.op(9, "invoke", "transfer", {"from": 1, "to": 2, "amount": i + 1})
        s.op(9, "ok", "transfer", {"from": 1, "to": 2, "amount": i + 1})
    for r in reads:
        s.op(0, "invoke", "read").op(0, "ok", "read", r)
    return s.flat("bank")


def read_event(h: H.FlatHistory, k: int) -> int:
    """Position of the k-th :ok read of h."""
    return int(np.flatnonzero((h.type == H.T_OK) & (h.f == H.F_READ))[k])


# the :index of read k of _bank(reads) without transfers is 2k + 1
BANK_OUTCOME_READS = [
    ZERO,                                   # 0 ok
    {**ZERO, 9: 0},                         # 1 unexpected-key (1)
    {**ZERO, 3: None},                      # 2 nil-balance (1)
    {**ZERO, 1: 5},                         # 3 wrong-total (5)
    {**ZERO, 1: -4, 2: 4},                  # 4 negative-value (4) when negatives are forbidden, else ok
]
BANK_OUTCOME_TYPES = [0, 1, 2, 3, 4]

# precedence: unexpected-key > nil-balance > wrong-total > negative-value, then ties
BANK_PRECEDENCE_READS = [
    {**ZERO, 1: None, 2: -3, 9: 1, 10: 2},  # 0 unexpected (2), also nil, wrong-total, negative
    {**ZERO, 1: None, 2: -3, 3: 10},        # 1 nil (1), also wrong-total, negative
    {**ZERO, 1: -3, 2: 10},                 # 2 wrong-total (|7|), also negative
    {**ZERO, 1: -3, 2: 3},                  # 3 negative (3)
    {**ZERO, 4: None, 11: 0, 12: 0},        # 4 unexpected (2): ties read 0
    {**ZERO, 5: None},                      # 5 nil (1): ties read 1
    {**ZERO, 1: 4, 2: 3},                   # 6 wrong-total (|7|): ties read 2, equal lowest and highest total
    {**ZERO, 3: -3, 4: 3},                  # 7 negative (3): ties read 3
    {**ZERO, 1: -2, 2: 2},                  # 8 negative (2): less bad
]
BANK_PRECEDENCE_TYPES = [1, 2, 3, 4, 1, 2, 3, 4, 4]


def bank_outcomes() -> H.FlatHistory:
    return _bank(BANK_OUTCOME_READS)


def bank_precedence() -> H.FlatHistory:
    return _bank(BANK_PRECEDENCE_READS)


FLOAT_TIE_TOTAL = 7
FLOAT_TIE_DIFFS = (100_000_000, 100_000_001)


def bank_float_tie() -> H.FlatHistory:
    """total_amount 7 and two wrong totals 7 + 1e8 (earlier) and 7 + 1e8 + 1 (later): their ratios to 7 differ as
    doubles but are equal after (float ...), so the earlier read is the worst."""
    return _bank([{**ZERO, 1: FLOAT_TIE_TOTAL + d} for d in FLOAT_TIE_DIFFS])


def bank_extremes() -> H.FlatHistory:
    """Balances at INT32_MAX and INT32_MIN + 1 (totals far outside int32), the nil sentinel, and reads whose payload
    length is odd (a trailing id without a balance) or 1."""
    reads = [{a: INT32_MAX for a in ACCOUNTS}, {a: INT32_MIN + 1 for a in ACCOUNTS},
             {**ZERO, 1: INT32_MAX, 2: INT32_MIN + 1}, {**ZERO, 1: None, 2: INT32_MAX},
             {**ZERO, 1: INT32_MIN + 1, 2: INT32_MAX}, {**ZERO, 1: -5, 2: 5}, {**ZERO, 9: 3}, ZERO]
    h = _bank(reads, transfers=2)
    h.payload_len[read_event(h, 6)] -= 1     # ... 8 0 9 -> the unexpected id 9 has no balance: ignored
    h.payload_len[read_event(h, 5)] = 1      # a lone id
    return h


def bank_many(n_reads: int = 1500, seed: int = 0) -> H.FlatHistory:
    """n_reads reads (>= 4 blocks of 256) drawn from a small palette, so equal badness and equal extreme totals recur
    in different blocks and bk_scan's atomics race across them."""
    rng = np.random.default_rng(seed)
    reads = []
    for _ in range(n_reads):
        r = dict(ZERO)
        kind = rng.integers(0, 6)
        a = int(rng.integers(1, 9))
        if kind == 1:
            r[9 + int(rng.integers(0, 2))] = 0
        elif kind == 2:
            r[a] = None
        elif kind == 3:
            r[a] = int(rng.choice([-3, -1, 2, 5]))
        elif kind == 4:
            b = a % 8 + 1
            r[a], r[b] = -int(rng.integers(1, 3)), 0
            r[b] = -r[a]
        reads.append(r)
    return _bank(reads)


def bank_no_reads() -> H.FlatHistory:
    return _bank([], transfers=3)


# name -> (builder, total_amount)
BANK_SHAPES = {
    "outcomes": (bank_outcomes, 0), "outcomes-total": (bank_outcomes, 5),
    "precedence": (bank_precedence, 0), "precedence-total": (bank_precedence, 7),
    "float-tie": (bank_float_tie, FLOAT_TIE_TOTAL), "extremes": (bank_extremes, 0), "extremes-total": (bank_extremes, 3),
    "many": (bank_many, 0), "many-total": (bank_many, 2), "no-reads": (bank_no_reads, 0),
}


# =====================================================================================================================
# partition and ledger balances
# =====================================================================================================================
PARTITION_SIZES = (1, 255, 256, 257, 2 ** 20 + 1)
SPECIAL_KEYS = np.array([INT64_MIN, INT64_MAX, -1, 0], np.int64)


def partition_keys(n: int, kind: str, seed: int = 0) -> np.ndarray:
    """Event keys: "specials" (INT64_MIN, INT64_MAX, -1, 0 and a few others, repeated), "equal" (one key), "distinct"
    (every key different, the specials among them)."""
    rng = np.random.default_rng(seed)
    if kind == "equal":
        return np.full(n, -1, np.int64)
    if kind == "specials":
        palette = np.concatenate([SPECIAL_KEYS, np.array([1, -2, INT64_MIN + 1, INT64_MAX - 1], np.int64)])
        return rng.choice(palette, size=n).astype(np.int64)
    assert kind == "distinct"
    k = np.unique(rng.integers(INT64_MIN, INT64_MAX, size=n + 8, dtype=np.int64))
    k = np.setdiff1d(k, SPECIAL_KEYS)[:max(0, n - 4)]
    k = np.concatenate([SPECIAL_KEYS[:min(4, n)], k])
    rng.shuffle(k)
    return k.astype(np.int64)


def wide_balances():
    """(credits, debits) whose differences leave int32 (no int64 overflow), with the int32-truncated expectation."""
    c = np.array([2 ** 31, 0, 2 ** 40 + 5, -(2 ** 40), INT32_MAX, 0, 2 ** 32, 2 ** 61 + 3, 7], np.int64)
    d = np.array([0, 2 ** 31 + 1, 3, 2 ** 40, -1, INT32_MIN, 0, -(2 ** 61), 9], np.int64)
    expect = np.array([((int(x) - int(y) + 2 ** 31) % 2 ** 32) - 2 ** 31 for x, y in zip(c, d)], np.int32)
    return c, d, expect
