"""Stored ledger and set-full histories: seeded op maps, and the EDN text Jepsen's store writes for them.

`ledger_ops` turns a ledger-lookups FlatHistory (`synth.generate_ledger_lookups`) back into the op maps a ledger test
records (tests/ledger.clj:27-87): transfers as [[:t id {:debit-acct d :credit-acct c :amount a}]], reads as
[[:r account {:debits-posted d :credits-posted c}] ...], lookups as [[:l-t id {...}] ...], with the final phase's
:final? reads and lookups.  `write_edn` writes op maps the way the store writes history.edn: one
`#jepsen.history.Op{...}` per line (or one vector of op maps), keywords for keyword-like strings, EDN strings for the
rest.  Tests and `scripts/edn_read_bench.py` use both to feed the device reader (`Context.read_ledger_edn`) and the
Python path (`edn.read_history` + `history.flatten_ops`) the same bytes.

`set_ops` does the same for a keyed set history (`synth.config_c4` and friends): the op maps a set-full test records
(workloads/set_full.clj:29-45, 107-134), for `Context.read_set_edn` and `edn.read_history(text, independent=True)`.
"""
from __future__ import annotations

import re
from typing import Any, Iterable, Mapping

import numpy as np

from . import synth
from .history import (F_ADD, F_LOOKUP, F_READ, F_TRANSFER, FLAG_FINAL, T_INFO, T_INVOKE, T_OK, TRANSFER_RECORD,
                      FlatHistory, transfer_id)

TYPE_NAME = {0: "invoke", 1: "ok", 2: "fail", 3: "info"}
_KEYWORD = re.compile(r"[A-Za-z*+!_?<>=-][A-Za-z0-9*+!_?<>=./-]*\Z")


def ledger_ops(h: FlatHistory, nemesis_every: int = 0) -> list[dict]:
    """The op maps of a ledger-lookups history: `flatten_ops(ledger_ops(h), "ledger-lookups")` has h's arrays.  A
    completion repeats its invocation's value, except an :ok read (the counters it saw) and an :ok lookup (the records
    it returned; [] when it found none, which takes its tag from the pending invoke).  nemesis_every > 0 inserts a
    nemesis op (process :nemesis, no :index, nested values and strings holding brackets, quotes and backslashes) before
    every nemesis_every-th client op."""
    n = h.n_events
    accounts = sorted({int(k) // 2 for e in range(n) if h.f[e] == F_READ and h.payload_len[e] > 0
                       for k in h.payload[h.payload_off[e]:h.payload_off[e] + h.payload_len[e]:3]})
    completion: dict[int, int] = {}     # lookup invoke -> its completion
    open_lookup: dict[int, int] = {}
    for e in range(n):
        if h.f[e] == F_LOOKUP:
            if h.type[e] == T_INVOKE:
                open_lookup[int(h.process[e])] = e
            else:
                completion[open_lookup.pop(int(h.process[e]))] = e
    pending: dict[int, list] = {}
    shared: dict[bytes, list] = {}      # lookups returning the same records share one value list
    ops: list[dict] = []
    for e in range(n):
        p, t = int(h.process[e]), int(h.type[e])
        pl = h.payload[h.payload_off[e]:h.payload_off[e] + max(int(h.payload_len[e]), 0)]
        if h.f[e] == F_TRANSFER:
            if t == T_INVOKE:
                value = [["t", transfer_id(r[0], r[1]), {"debit-acct": int(r[2]), "credit-acct": int(r[3]),
                                                         "amount": int(r[4])}]
                         for r in pl.reshape(-1, TRANSFER_RECORD)]
                pending[p] = value
            else:
                value = pending.pop(p)
        elif h.f[e] == F_READ:
            if t == T_OK:
                seen: dict[int, dict] = {}
                for k, lo, hi in pl.reshape(-1, 3):
                    name = "credits-posted" if k & 1 else "debits-posted"
                    seen.setdefault(int(k) // 2, {})[name] = transfer_id(lo, hi)
                value = [["r", a, {"debits-posted": m.get("debits-posted"), "credits-posted": m.get("credits-posted")}]
                         for a, m in seen.items()]
            else:
                value = [["r", a, None] for a in accounts]
        else:
            key = pl.tobytes()
            if t == T_OK and key not in shared:
                shared[key] = [["l-t", transfer_id(r[0], r[1]), {"debit-acct": int(r[2]), "credit-acct": int(r[3]),
                                                                  "amount": int(r[4])}]
                               for r in pl.reshape(-1, TRANSFER_RECORD)]
            recs = shared.get(key)
            if t == T_INVOKE:
                c = completion.get(e)
                cpl = (h.payload[h.payload_off[c]:h.payload_off[c] + max(int(h.payload_len[c]), 0)]
                       if c is not None else np.zeros(0, np.int32))
                value = [["l-t", transfer_id(r[0], r[1]), None] for r in cpl.reshape(-1, TRANSFER_RECORD)]
                value = value or [["l-t", 1, None]]
                pending[p] = value
            elif t == T_OK:
                value = recs
                pending.pop(p, None)
            else:
                value = pending.pop(p)
        op = {"index": int(h.index[e]), "time": int(h.time_ns[e]), "type": TYPE_NAME[t], "process": p, "f": "txn",
              "value": value}
        if h.flags[e] & FLAG_FINAL:
            op["final?"] = True
        if nemesis_every > 0 and e % nemesis_every == nemesis_every - 1:
            ops.append(_nemesis_op(len(ops), int(h.time_ns[e])))
        ops.append(op)
    return ops


def _nemesis_op(k: int, time: int) -> dict:
    start = k % 2 == 0
    return {"time": time, "type": "info", "process": "nemesis", "f": "start-partition" if start else "stop-partition",
            "value": {"n1": ["n2", "n3"], "note": 'cut ]} "n1" \\ off', "nodes": frozenset({"n4", "n5"})}
            if start else "network healed"}


def generate_ledger_ops(spec: synth.SynthSpec, p_lookup: float = 0.0, nemesis_every: int = 0,
                        **mutations) -> list[dict]:
    """Seeded ledger op maps: `ledger_ops(synth.generate_ledger_lookups(spec, p_lookup, **mutations))` — :info and :fail
    transfers from spec.p_info, mid-run lookups from p_lookup, and the final phase (one :final? read, then one :final?
    lookup per client returning every committed transfer) when spec.final_reads."""
    return ledger_ops(synth.generate_ledger_lookups(spec, p_lookup=p_lookup, **mutations), nemesis_every)


def set_ops(h: FlatHistory, nemesis_every: int = 0) -> list[dict]:
    """The op maps of a keyed set history, in history order across keys (by :index): `flatten_ops(
    edn.read_history(write_edn(set_ops(h)), independent=True), "set")` has h's events, keys and read payloads.  An add is
    [k id] on its invoke and completion; a read invoke is [k nil] and an :ok read [k #{ids}]; an :info completion
    repeats its invoke's value with :error :timeout; the final reads carry :final? true.  nemesis_every > 0 inserts a
    nemesis op before every nemesis_every-th client op, as `ledger_ops` does."""
    key = np.repeat(h.key_ids, np.diff(h.shard_off))
    ops: list[dict] = []
    for c, e in enumerate(np.argsort(h.index, kind="stable")):
        t, k = int(h.type[e]), int(key[e])
        if h.f[e] == F_ADD:
            f, value = "add", (k, int(h.a[e]))
        elif h.f[e] == F_READ:
            pl = h.payload[h.payload_off[e]:h.payload_off[e] + max(int(h.payload_len[e]), 0)]
            f, value = "read", (k, frozenset(int(x) for x in pl) if t == T_OK else None)
        else:
            raise ValueError(f"event {e}: not a set-full :add or :read")
        op = {"index": int(h.index[e]), "time": int(h.time_ns[e]), "type": TYPE_NAME[t], "process": int(h.process[e]),
              "f": f, "value": value}
        if t == T_INFO:
            op["error"] = "timeout"
        if h.flags[e] & FLAG_FINAL:
            op["final?"] = True
        if nemesis_every > 0 and c % nemesis_every == nemesis_every - 1:
            ops.append(_nemesis_op(len(ops), int(h.time_ns[e])))
        ops.append(op)
    return ops


def generate_set_ops(spec: synth.SynthSpec, nemesis_every: int = 0) -> list[dict]:
    """Seeded set-full op maps: `set_ops(synth.generate(spec))` for a spec of model "set" (e.g. the shapes of
    synth.config_c1 and config_c4)."""
    if spec.model != "set":
        raise ValueError(f"a set-full history needs a spec of model 'set', not {spec.model!r}")
    return set_ops(synth.generate(spec), nemesis_every)


def _value(v: Any, memo: dict | None = None) -> str:
    if memo is not None and isinstance(v, list) and len(v) > 64:
        hit = memo.get(id(v))
        if hit is None or hit[0] is not v:
            hit = memo[id(v)] = (v, _value(v))
        return hit[1]
    if v is None:
        return "nil"
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, str):
        if _KEYWORD.match(v):
            return ":" + v
        return '"' + v.replace("\\", "\\\\").replace('"', '\\"') + '"'
    if isinstance(v, (list, tuple)):
        return "[" + " ".join(_value(x) for x in v) + "]"
    if isinstance(v, (set, frozenset)):
        return "#{" + " ".join(_value(x) for x in sorted(v)) + "}"
    if isinstance(v, Mapping):
        return "{" + ", ".join(f"{_value(k)} {_value(x)}" for k, x in v.items()) + "}"
    return str(int(v))


_FIRST = ("index", "time", "type", "process", "f", "value")


def op_line(op: Mapping[str, Any], tagged: bool = True, memo: dict | None = None) -> str:
    """One op map as the store writes it: the record's fields first (:index :time :type :process :f :value), then the
    rest in their order."""
    keys = [k for k in _FIRST if k in op] + [k for k in op if k not in _FIRST]
    body = "{" + ", ".join(f":{k} {_value(op[k], memo)}" for k in keys) + "}"
    return ("#jepsen.history.Op" + body) if tagged else body


def write_edn(ops: Iterable[Mapping[str, Any]], vector: bool = False, tagged: bool = True,
              newline: str = "\n") -> bytes:
    """history.edn bytes of `ops`: one op per line, or (vector=True) one top-level vector holding them."""
    memo: dict = {}   # a long value shared by several ops (the final lookups' records) is formatted once
    lines = [op_line(op, tagged, memo) for op in ops]
    if vector:
        text = "[" + newline.join(lines) + "]" + newline
    else:
        text = newline.join(lines) + newline
    return text.encode()
