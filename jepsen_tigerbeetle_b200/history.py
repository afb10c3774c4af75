"""Flat struct-of-arrays history IR and the op-map flattener.

This is the tested Python twin of the Clojure/JNI glue (`clj/jtb/checker.clj`): it turns a Jepsen
history (a vector of op maps) into the `jtb_history` arrays declared in `include/jtb_check.h`.

Op shapes accepted (reference file:line):
  * set-full:   {:type :invoke :f :add  :value [k v]}            set_full.clj:29-31
                {:type :ok     :f :read :value [k #{ids}]}       set_full.clj:128-134
                {:type :info   :error :timeout}                  set_full.clj:107-110,122-125
                {:final? true}                                   set_full.clj:45
  * ledger:     {:f :txn :value [[:r id {:credits-posted c :debits-posted d}] ...]}
                {:f :txn :value [[:t id {:debit-acct d :credit-acct c :amount a}]]}
                {:f :txn :value [[:l-t ...]]}  (dropped; kept by 'ledger-lookups')  tests/ledger.clj:27-62,89-114
  * bank (jepsen.tests.bank): {:f :read :value {id bal}} / {:f :transfer :value {:from :to :amount}}
  * register / cas-register (knossos.model): :read v|nil, :write v, :cas [old new]

`independent/tuple` values ([k v]) are split per key into CSR shards (jepsen.independent/subhistory,
SURVEY A.2): ops whose value is not a tuple (nemesis etc.) have process < 0 here and are ignored by
all checkers, so they are simply not replicated into shards.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field
from typing import Any, Iterable, Mapping, Sequence

import numpy as np

# ---- constants mirrored from include/jtb_check.h ------------------------------------------------
VALID, UNKNOWN, INVALID = 0, 1, 2
T_INVOKE, T_OK, T_FAIL, T_INFO = 0, 1, 2, 3
F_READ, F_WRITE, F_CAS, F_ADD, F_TRANSFER, F_LOOKUP = 0, 1, 2, 3, 4, 5
NIL = -(2 ** 31)
FLAG_FINAL = 1
MODEL_REGISTER, MODEL_CAS_REGISTER, MODEL_SET, MODEL_BANK = 0, 1, 2, 3
MAX_ACCOUNTS = 8

TYPE_CODE = {"invoke": T_INVOKE, "ok": T_OK, "fail": T_FAIL, "info": T_INFO}
VERDICT_NAME = {VALID: True, UNKNOWN: "unknown", INVALID: False}


def merge_valid(verdicts: Iterable[int]) -> int:
    """jepsen.checker/merge-valid: false dominates :unknown dominates true (SURVEY A.2)."""
    out = VALID
    for v in verdicts:
        out = max(out, int(v))
    return out


@dataclass
class FlatHistory:
    """Struct-of-arrays history (see `jtb_history` in include/jtb_check.h)."""

    type: np.ndarray
    f: np.ndarray
    flags: np.ndarray
    process: np.ndarray
    index: np.ndarray
    time_ns: np.ndarray
    a: np.ndarray
    b: np.ndarray
    c: np.ndarray
    payload_off: np.ndarray
    payload_len: np.ndarray
    payload: np.ndarray
    shard_off: np.ndarray
    key_ids: np.ndarray
    meta: dict = field(default_factory=dict)

    @property
    def n_events(self) -> int:
        return int(self.type.shape[0])

    @property
    def n_shards(self) -> int:
        return int(self.shard_off.shape[0] - 1)

    def validate(self) -> None:
        n = self.n_events
        for name, dt in (("type", np.uint8), ("f", np.uint8), ("flags", np.uint8),
                         ("process", np.int32), ("index", np.int32), ("time_ns", np.int64),
                         ("a", np.int32), ("b", np.int32), ("c", np.int32),
                         ("payload_off", np.int64), ("payload_len", np.int32)):
            arr = getattr(self, name)
            assert arr.dtype == dt and arr.shape == (n,) and arr.flags.c_contiguous, name
        assert self.payload.dtype == np.int32 and self.payload.flags.c_contiguous
        assert self.shard_off.dtype == np.int64 and self.shard_off[0] == 0
        assert self.shard_off[-1] == n and np.all(np.diff(self.shard_off) >= 0)
        assert self.key_ids.dtype == np.int64 and self.key_ids.shape == (self.n_shards,)

    def select_shards(self, shards: Sequence[int]) -> "FlatHistory":
        """The sub-history made of the given shards (in that order) — what one rank of a multi-GPU
        check receives.  Events keep their original :index, so witnesses stay globally meaningful."""
        shards = [int(s) for s in shards]
        lo = self.shard_off[shards] if shards else np.zeros(0, np.int64)
        hi = self.shard_off[[s + 1 for s in shards]] if shards else np.zeros(0, np.int64)
        counts = (hi - lo).astype(np.int64)
        ev = (np.concatenate([np.arange(a, b, dtype=np.int64) for a, b in zip(lo, hi)])
              if shards else np.zeros(0, np.int64))
        plen = np.maximum(self.payload_len[ev], 0).astype(np.int64)
        new_off = np.zeros(ev.shape[0], np.int64)
        if ev.shape[0]:
            np.cumsum(plen[:-1], out=new_off[1:])
        total = int(plen.sum())
        payload = np.zeros(total, np.int32)
        if total:
            # gather payload ranges: index = old_off[event] + position inside the event's payload
            rep = np.repeat(np.arange(ev.shape[0]), plen)
            inner = np.arange(total, dtype=np.int64) - np.repeat(new_off, plen)
            payload = self.payload[self.payload_off[ev][rep] + inner].astype(np.int32)
        shard_off = np.zeros(len(shards) + 1, np.int64)
        np.cumsum(counts, out=shard_off[1:])
        return FlatHistory(self.type[ev], self.f[ev], self.flags[ev], self.process[ev], self.index[ev],
                           self.time_ns[ev], self.a[ev], self.b[ev], self.c[ev], new_off,
                           self.payload_len[ev], payload, shard_off,
                           self.key_ids[shards].astype(np.int64) if shards else np.zeros(0, np.int64),
                           dict(self.meta))

    def shard(self, s: int) -> "FlatHistory":
        """A single-shard view (copy) — `independent/subhistory` for key s."""
        lo, hi = int(self.shard_off[s]), int(self.shard_off[s + 1])
        sl = slice(lo, hi)
        plen = np.maximum(self.payload_len[sl], 0).astype(np.int64)
        new_off = np.zeros(hi - lo, dtype=np.int64)
        if hi > lo:
            np.cumsum(plen[:-1], out=new_off[1:])
        chunks = [self.payload[int(o):int(o) + int(l)] for o, l in zip(self.payload_off[sl], plen)]
        payload = np.concatenate(chunks) if chunks else np.zeros(0, np.int32)
        return FlatHistory(self.type[sl].copy(), self.f[sl].copy(), self.flags[sl].copy(),
                           self.process[sl].copy(), self.index[sl].copy(), self.time_ns[sl].copy(),
                           self.a[sl].copy(), self.b[sl].copy(), self.c[sl].copy(), new_off,
                           self.payload_len[sl].copy(), payload.astype(np.int32),
                           np.array([0, hi - lo], np.int64), self.key_ids[s:s + 1].copy(),
                           dict(self.meta))


def concat_keys(parts: Sequence[FlatHistory]) -> FlatHistory:
    """Several single-key histories as ONE keyed history (shard s = parts[s], key id s + 1) — the shape
    `independent/checker` sees when every ledger/key has its own sub-history."""
    cat = lambda name: np.concatenate([getattr(p, name) for p in parts])  # noqa: E731
    poff, base = [], 0
    for p in parts:
        poff.append(p.payload_off + base)
        base += int(p.payload.shape[0])
    shard_off = np.zeros(len(parts) + 1, np.int64)
    np.cumsum([p.n_events for p in parts], out=shard_off[1:])
    return FlatHistory(cat("type"), cat("f"), cat("flags"), cat("process"), cat("index"), cat("time_ns"),
                       cat("a"), cat("b"), cat("c"), np.concatenate(poff).astype(np.int64), cat("payload_len"),
                       cat("payload"), shard_off, np.arange(1, len(parts) + 1, dtype=np.int64),
                       dict(parts[0].meta) if parts else {})


class CHistory(ctypes.Structure):
    """ctypes image of `struct jtb_history`."""

    _fields_ = [
        ("n_events", ctypes.c_int64),
        ("type", ctypes.c_void_p), ("f", ctypes.c_void_p), ("flags", ctypes.c_void_p),
        ("process", ctypes.c_void_p), ("index", ctypes.c_void_p), ("time_ns", ctypes.c_void_p),
        ("a", ctypes.c_void_p), ("b", ctypes.c_void_p), ("c", ctypes.c_void_p),
        ("payload_off", ctypes.c_void_p), ("payload_len", ctypes.c_void_p),
        ("payload", ctypes.c_void_p), ("n_payload", ctypes.c_int64),
        ("n_shards", ctypes.c_int32),
        ("shard_off", ctypes.c_void_p), ("key_ids", ctypes.c_void_p),
    ]


class CModel(ctypes.Structure):
    """ctypes image of `struct jtb_model`."""

    _fields_ = [
        ("kind", ctypes.c_int32), ("init_value", ctypes.c_int32), ("n_accounts", ctypes.c_int32),
        ("account_ids", ctypes.c_int32 * MAX_ACCOUNTS),
        ("init_balance", ctypes.c_int32 * MAX_ACCOUNTS),
        ("negative_balances_ok", ctypes.c_int32),
    ]


def as_c_history(h: FlatHistory) -> CHistory:
    """Borrow the numpy buffers of `h` (caller keeps `h` alive for the duration of the call)."""
    h.validate()
    p = lambda arr: arr.ctypes.data  # noqa: E731
    return CHistory(h.n_events, p(h.type), p(h.f), p(h.flags), p(h.process), p(h.index),
                    p(h.time_ns), p(h.a), p(h.b), p(h.c), p(h.payload_off), p(h.payload_len),
                    p(h.payload), int(h.payload.shape[0]), h.n_shards, p(h.shard_off),
                    p(h.key_ids))


def make_model(kind: int, init_value: int = NIL, accounts: Sequence[int] = (),
               init_balance: Sequence[int] | None = None,
               negative_balances_ok: bool = True) -> CModel:
    m = CModel()
    m.kind = kind
    m.init_value = init_value
    accounts = list(accounts)
    if len(accounts) > MAX_ACCOUNTS:
        raise ValueError(f"at most {MAX_ACCOUNTS} accounts supported")
    m.n_accounts = len(accounts)
    for i, acct in enumerate(accounts):
        m.account_ids[i] = int(acct)
        m.init_balance[i] = int(init_balance[i]) if init_balance is not None else 0
    m.negative_balances_ok = 1 if negative_balances_ok else 0
    return m


# ---- builder ------------------------------------------------------------------------------------
class _Builder:
    def __init__(self) -> None:
        self.rows: list[tuple] = []     # (key, type, f, flags, process, index, time, a, b, c, payload|None)

    def add(self, key, type_, f, flags, process, index, time, a=0, b=0, c=0, payload=None):
        self.rows.append((key, type_, f, flags, process, index, time, a, b, c, payload))

    def build(self, meta: dict | None = None) -> FlatHistory:
        keys = sorted({r[0] for r in self.rows}, key=lambda k: (k is None, k))
        if not keys:
            keys = [None]
        by_key: dict[Any, list[tuple]] = {k: [] for k in keys}
        for r in self.rows:
            by_key[r[0]].append(r)
        n = len(self.rows)
        typ = np.zeros(n, np.uint8); f = np.zeros(n, np.uint8); flags = np.zeros(n, np.uint8)
        proc = np.zeros(n, np.int32); idx = np.zeros(n, np.int32); t = np.zeros(n, np.int64)
        a = np.zeros(n, np.int32); b = np.zeros(n, np.int32); c = np.zeros(n, np.int32)
        poff = np.zeros(n, np.int64); plen = np.zeros(n, np.int32)
        payload: list[int] = []
        shard_off = [0]
        i = 0
        for k in keys:
            for r in by_key[k]:
                (_, typ[i], f[i], flags[i], proc[i], idx[i], t[i], a[i], b[i], c[i], pl) = r
                poff[i] = len(payload)
                if pl is None:
                    plen[i] = -1
                else:
                    plen[i] = len(pl)
                    payload.extend(int(x) for x in pl)
                i += 1
            shard_off.append(i)
        key_ids = np.array([(-1 if k is None else int(k)) for k in keys], np.int64)
        return FlatHistory(typ, f, flags, proc, idx, t, a, b, c, poff, plen,
                           np.array(payload, np.int32), np.array(shard_off, np.int64), key_ids,
                           dict(meta or {}))


def _kw(x: Any) -> Any:
    """Accept Clojure-style keywords spelled ':add' as well as 'add'."""
    if isinstance(x, str) and x.startswith(":"):
        return x[1:]
    return x


def _get(m: Mapping, *names: str, default=None):
    for nm in names:
        if nm in m:
            return m[nm]
        if ":" + nm in m:
            return m[":" + nm]
    return default


def is_tuple(v: Any) -> bool:
    """`independent/tuple?` — we represent tuples as Python tuples of length 2 (lists are plain
    vectors, e.g. a :cas [old new])."""
    return isinstance(v, tuple) and len(v) == 2


def flatten_ops(ops: Sequence[Mapping[str, Any]], model: str) -> FlatHistory:
    """Flatten a Jepsen history (sequence of op maps) for `model` in
    {'register','cas-register','set','bank','ledger-counters','ledger-lookups'}.

    'ledger-counters' keeps what 'bank' folds into a balance: every account of a ledger :r read becomes two
    (key, value_lo, value_hi) triples, key = 2*account + field (0 debits-posted, 1 credits-posted), the input of the
    monotonic-key and counter-bounds checks.  Like ledger->bank it keeps only the first [:t ...] of a transfer txn;
    meta["multi_transfer_txns"] counts the transfer txns (at their invocation) that had more than one micro-op, since
    the counter-bounds check would miss the others' amounts.

    'ledger-lookups' is 'ledger-counters' plus the transfer-lookup check's evidence: a transfer invoke also carries one
    record (id_lo, id_hi, debit, credit, amount) per [:t ...] micro-op (a multi-transfer txn is kept whole; a, b, c
    stay the first micro-op's), and every [:l-t ...] op becomes an F_LOOKUP event whose :ok payload is the returned
    records in the same layout (nil on the invoke, :info and :fail).  An :ok lookup with an empty value takes its tag
    from its process's pending invoke.

    For 'bank', ledger-form :txn ops are first mapped by `ledger->bank` (tests/ledger.clj:89-114);
    stock jepsen.tests.bank {:from :to :amount} spelling is accepted too (SURVEY App. D).
    """
    model = _kw(model)
    bld = _Builder()
    multi_transfer = 0
    pending_tag: dict = {}   # ledger-lookups: process -> the txn tag of its pending invoke
    for pos, op in enumerate(ops):
        type_ = TYPE_CODE[_kw(_get(op, "type"))]
        process = _get(op, "process")
        index = _get(op, "index", default=pos)
        time = int(_get(op, "time", default=pos))
        flags = FLAG_FINAL if _get(op, "final?", default=False) else 0
        value = _get(op, "value")
        f = _kw(_get(op, "f"))
        if not isinstance(process, (int, np.integer)) or isinstance(process, bool):
            continue  # :nemesis etc.: ignored by every checker on this path
        key = None
        if is_tuple(value):
            key, value = value
        if model in ("register", "cas-register"):
            if f == "read":
                bld.add(key, type_, F_READ, flags, process, index, time,
                        a=NIL if value is None else int(value))
            elif f == "write":
                bld.add(key, type_, F_WRITE, flags, process, index, time, a=int(value))
            elif f == "cas":
                old, new = value
                bld.add(key, type_, F_CAS, flags, process, index, time, a=int(old), b=int(new))
            else:
                raise ValueError(f"unknown :f {f!r} for model {model}")
        elif model == "set":
            if f == "add":
                if value is None:
                    continue  # [nil nil] add-ok of a rejected account (SURVEY App. D): skipped
                bld.add(key, type_, F_ADD, flags, process, index, time, a=int(value))
            elif f == "read":
                pl = None if value is None else [int(x) for x in value]
                if pl is not None and not isinstance(value, (list, tuple)):
                    pl = sorted(pl)  # sets / sorted-sets: canonical order
                bld.add(key, type_, F_READ, flags, process, index, time, payload=pl)
            else:
                raise ValueError(f"unknown :f {f!r} for model set")
        elif model == "bank":
            if f == "txn":  # ledger form -> ledger->bank
                first = value[0]
                tag = _kw(first[0])
                if tag == "r":
                    if type_ == T_OK:
                        pl: list[int] = []
                        for (_r, acct, amounts) in value:
                            pl.append(int(acct))
                            if amounts is None:
                                pl.append(NIL)
                            else:
                                cp = _get(amounts, "credits-posted")
                                dp = _get(amounts, "debits-posted")
                                pl.append(NIL if cp is None or dp is None else int(cp) - int(dp))
                        bld.add(key, type_, F_READ, flags, process, index, time, payload=pl)
                    else:
                        bld.add(key, type_, F_READ, flags, process, index, time, payload=None)
                elif tag == "t":
                    (_t, _id, tv) = first
                    bld.add(key, type_, F_TRANSFER, flags, process, index, time,
                            a=int(_get(tv, "amount")), b=int(_get(tv, "debit-acct")),
                            c=int(_get(tv, "credit-acct")))
                elif tag == "l-t":
                    continue  # dropped by ledger->bank (tests/ledger.clj:110-111)
                else:
                    raise ValueError(f"unknown txn micro-op {tag!r}")
            elif f == "read":
                pl = None
                if value is not None and type_ == T_OK:
                    pl = []
                    for acct, bal in value.items():
                        pl.append(int(acct))
                        pl.append(NIL if bal is None else int(bal))
                bld.add(key, type_, F_READ, flags, process, index, time, payload=pl)
            elif f == "transfer":
                d = _get(value, "debit-acct", "from")
                cr = _get(value, "credit-acct", "to")
                bld.add(key, type_, F_TRANSFER, flags, process, index, time,
                        a=int(_get(value, "amount")), b=int(d), c=int(cr))
            else:
                raise ValueError(f"unknown :f {f!r} for model bank")
        elif model == "ledger-counters":
            if f != "txn":
                raise ValueError(f"unknown :f {f!r} for model ledger-counters")
            tag = _kw(value[0][0])
            if tag == "r":
                bld.add(key, type_, F_READ, flags, process, index, time,
                        payload=_counter_triples(value, index) if type_ == T_OK else None)
            elif tag == "t":
                (_t, _id, tv) = value[0]
                multi_transfer += type_ == T_INVOKE and len(value) > 1
                bld.add(key, type_, F_TRANSFER, flags, process, index, time,
                        a=int(_get(tv, "amount")), b=int(_get(tv, "debit-acct")),
                        c=int(_get(tv, "credit-acct")))
            elif tag == "l-t":
                continue  # dropped, as ledger->bank drops it (tests/ledger.clj:110-111)
            else:
                raise ValueError(f"unknown txn micro-op {tag!r}")
        elif model == "ledger-lookups":
            if f != "txn":
                raise ValueError(f"unknown :f {f!r} for model ledger-lookups")
            if value:
                tag = _kw(value[0][0])
            elif type_ != T_INVOKE and process in pending_tag:
                tag = pending_tag[process]   # an empty :ok lookup: value[0][0] does not exist
            else:
                raise ValueError(f"op {index}: a txn without micro-ops")
            if type_ == T_INVOKE:
                pending_tag[process] = tag
            else:
                pending_tag.pop(process, None)
            if tag == "r":
                bld.add(key, type_, F_READ, flags, process, index, time,
                        payload=_counter_triples(value, index) if type_ == T_OK else None)
            elif tag == "t":
                (_t, _id, tv) = value[0]
                multi_transfer += type_ == T_INVOKE and len(value) > 1
                bld.add(key, type_, F_TRANSFER, flags, process, index, time,
                        a=int(_get(tv, "amount")), b=int(_get(tv, "debit-acct")),
                        c=int(_get(tv, "credit-acct")),
                        payload=_transfer_records(value, index) if type_ == T_INVOKE else None)
            elif tag == "l-t":
                bld.add(key, type_, F_LOOKUP, flags, process, index, time,
                        payload=_transfer_records(value or [], index) if type_ == T_OK else None)
            else:
                raise ValueError(f"unknown txn micro-op {tag!r}")
        else:
            raise ValueError(f"unknown model {model!r}")
    if model in ("ledger-counters", "ledger-lookups"):
        return bld.build({"model": model, "multi_transfer_txns": int(multi_transfer)})
    return bld.build({"model": model})


COUNTER_FIELDS = ("debits-posted", "credits-posted")   # field 0, field 1 of a ledger-counters key
MAX_COUNTER_ACCOUNT = 1 << 30


def counter_key(account: int, field: int) -> int:
    """The monotonic-key check's key of an account's counter: 2 * account + field (0 debits, 1 credits)."""
    return 2 * int(account) + int(field)


def _counter_triples(value, index) -> list[int]:
    """A ledger :r txn's accounts as (key, value_lo, value_hi) triples; an account with nil amounts (or a nil
    counter) is left out, which makes the read partial."""
    pl: list[int] = []
    for (_r, acct, amounts) in value:
        acct = int(acct)
        if not 0 <= acct < MAX_COUNTER_ACCOUNT:
            raise ValueError(f"op {index}: account {acct} is outside [0, 2^30)")
        if amounts is None:
            continue
        for field, name in enumerate(COUNTER_FIELDS):
            v = _get(amounts, name)
            if v is None:
                continue
            v = int(v)
            if not -(1 << 63) <= v < (1 << 63):
                raise ValueError(f"op {index}: {name} {v} of account {acct} does not fit in int64")
            u = v & 0xFFFFFFFFFFFFFFFF
            lo, hi = u & 0xFFFFFFFF, u >> 32
            pl.extend((counter_key(acct, field), lo - (1 << 32) if lo >= 1 << 31 else lo,
                       hi - (1 << 32) if hi >= 1 << 31 else hi))
    return pl


TRANSFER_RECORD = 5   # int32 per transfer record of the ledger-lookups form: id_lo, id_hi, debit, credit, amount


def _i32(x: int) -> int:
    return x - (1 << 32) if x >= 1 << 31 else x


def _transfer_records(value, index) -> list[int]:
    """The [:t id {...}] or [:l-t id {...}] micro-ops of a txn as (id_lo, id_hi, debit, credit, amount) records; a
    lookup micro-op without a transfer map (not found) is left out."""
    pl: list[int] = []
    for (_tag, tid, tv) in value:
        if tv is None:
            continue
        if tid is None:
            raise ValueError(f"op {index}: a transfer without an id")
        tid = int(tid)
        if not -(1 << 63) <= tid < (1 << 63):
            raise ValueError(f"op {index}: transfer id {tid} does not fit in int64")
        u = tid & 0xFFFFFFFFFFFFFFFF
        pl.extend((_i32(u & 0xFFFFFFFF), _i32(u >> 32), int(_get(tv, "debit-acct")), int(_get(tv, "credit-acct")),
                   int(_get(tv, "amount"))))
    return pl


def transfer_id(lo: int, hi: int) -> int:
    """The int64 id of a record's (id_lo, id_hi) pair."""
    u = ((int(hi) & 0xFFFFFFFF) << 32) | (int(lo) & 0xFFFFFFFF)
    return u - (1 << 64) if u >= 1 << 63 else u
