"""Host-side mirror of the reference's checker interface (the drop-in boundary, SURVEY §8(b)).

The reference composes `jepsen.checker/Checker`s — one method, `(check [this test history opts])`
returning a map with a mandatory `:valid?` in {true, false, :unknown}:

    src/tigerbeetle/workloads/set_full.clj:155-158
        (independent/checker (checker/compose {:set-full (checker/set-full {:linearizable? true})
                                               :read-all-invoked-adds (read-all-invoked-adds)}))
    src/tigerbeetle/tests/ledger.clj:363-367
        (checker/compose {:SI (checker opts) :plot ... :lookup-transfers ... :final-reads ... :unexpected-ops ...})

This module gives the same names, argument meaning and error behaviour in Python, backed ONLY by the
CUDA library (native.Context -> libjtb_check.so).  Result maps use the Jepsen key names without the
leading colon ("valid?", "lost-count", ...); `:unknown` is the string "unknown".

Histories may be given as Jepsen op maps (list of dicts) or as an already flattened FlatHistory.
"""
from __future__ import annotations

import traceback
from collections.abc import Mapping
from typing import Any

import numpy as np

from . import abi
from .history import (INVALID, MODEL_BANK, MODEL_CAS_REGISTER, MODEL_REGISTER, MODEL_SET, UNKNOWN,
                      VALID, VERDICT_NAME, COUNTER_FIELDS, FlatHistory, flatten_ops, make_model, merge_valid)
from .native import Context

_MODEL_KIND = {"register": MODEL_REGISTER, "cas-register": MODEL_CAS_REGISTER, "set": MODEL_SET,
               "bank": MODEL_BANK}
_CODE = {True: VALID, "unknown": UNKNOWN, False: INVALID}


def valid_code(v: Any) -> int:
    """:valid? value -> lattice code (true < :unknown < false)."""
    return _CODE[v if v in (True, False) else "unknown"]


def merge_valid_values(vals) -> Any:
    """jepsen.checker/merge-valid over :valid? values (SURVEY A.2)."""
    return VERDICT_NAME[merge_valid(valid_code(v) for v in vals)]


class Checker:
    """`jepsen.checker/Checker` protocol."""

    def check(self, test: Mapping[str, Any], history, opts: Mapping[str, Any] | None = None) -> dict:
        raise NotImplementedError


def check_safe(checker: Checker, test, history, opts=None) -> dict:
    """jepsen.checker/check-safe: a checker that throws yields {:valid? :unknown :error ...}."""
    try:
        return checker.check(test, history, opts or {})
    except Exception:  # noqa: BLE001 - mirrors (catch Throwable t ...)
        return {"valid?": "unknown", "error": traceback.format_exc()}


class StoredOp(Mapping):
    """One op map of a stored history.edn, given by its bytes [begin, end) and parsed (`edn.loads`) only when it is
    first read.  It equals the dict `edn.read_history` gives for that op, so a result holding the 40 MB final lookups of
    a large history costs nothing until someone reads them."""

    __slots__ = ("_data", "_begin", "_end", "_op")

    def __init__(self, data: bytes, begin: int, end: int) -> None:
        self._data, self._begin, self._end, self._op = data, int(begin), int(end), None

    @property
    def parsed(self) -> bool:
        return self._op is not None

    def _map(self) -> dict:
        if self._op is None:
            from .edn import loads
            self._op = loads(self._data[self._begin:self._end].decode())
        return self._op

    def __getitem__(self, key):
        return self._map()[key]

    def __iter__(self):
        return iter(self._map())

    def __len__(self) -> int:
        return len(self._map())

    def __repr__(self) -> str:
        return repr(self._op) if self._op is not None else f"StoredOp(bytes {self._begin}..{self._end})"


class _StoredHistory:
    """The bytes of a stored history.edn (a path or its bytes), the native.Context the device reads them on (None opens
    one on device 0 when the device is first needed), and the op maps of `edn.read_history` for the checkers that
    iterate it (parsed once, on first use, and cached)."""

    _independent = False   # read_history(..., independent=): whether 2-vector :values are [key value] tuples

    def __init__(self, path_or_bytes, ctx=None) -> None:
        if isinstance(path_or_bytes, (bytes, bytearray, memoryview)):
            self.data = bytes(path_or_bytes)
        else:
            with open(path_or_bytes, "rb") as fh:
                self.data = fh.read()
        self._ctx = ctx
        self._forms: dict[str, FlatHistory] = {}
        self._ops: list | None = None

    def _context(self):
        if self._ctx is None:
            from .native import Context
            self._ctx = Context(device=0)
        return self._ctx

    def ops(self) -> list:
        if self._ops is None:
            from .edn import read_history
            self._ops = read_history(self.data.decode(), independent=self._independent)
        return self._ops

    def __iter__(self):
        return iter(self.ops())

    def __len__(self) -> int:
        return len(self.ops())

    def __getitem__(self, i):
        return self.ops()[i]


class StoredLedgerHistory(_StoredHistory):
    """A stored ledger history.edn (a path or its bytes) that the ledger checks read on the GPU (K18, K19).

    `_flat` asks it for the "bank", "ledger-counters" or "ledger-lookups" form and gets the device reader's FlatHistory,
    read once per form and cached, instead of flattening op maps in Python.  The host checkers of a `ledger_checker()`
    compose (unexpected-ops, final-reads, lookup-transfers) and stats build their results from one device summary
    (`checks()`, K19), whose flagged ops are `StoredOp`s parsed only when read.  When the device refuses the file they
    iterate it instead: iterating yields the op maps of `edn.read_history` (parsed once, on first use, and cached).
    ctx: the native.Context to read on; None opens one on device 0 when the device is first needed."""

    def __init__(self, path_or_bytes, ctx=None) -> None:
        super().__init__(path_or_bytes, ctx)
        self._checks: dict | None = None

    def flat(self, form: str) -> FlatHistory:
        if form not in self._forms:
            self._forms[form] = self._context().read_ledger_edn(self.data, form)
        return self._forms[form]

    def checks(self) -> dict | None:
        """The device summary the host checkers use (`Context.ledger_edn_checks`), computed once; None when the device
        refused the file."""
        if self._checks is None:
            self._checks = self._context().ledger_edn_checks(self.data)
        return None if self._checks["refused"] else self._checks


class StoredSetHistory(_StoredHistory):
    """A stored set-full history.edn (a path or its bytes) that the set checks read on the GPU (K20).

    `_flat` asks it for the "set" form, which SetFull, ReadAllInvokedAdds, `independent_checker` and
    `linearizable({"model": "set"})` read, and gets the device reader's keyed FlatHistory (`Context.read_set_edn`), read
    once and cached, instead of flattening op maps in Python.  When the device refuses the file (`refused` then holds
    its reason), and for any other model, the op maps are flattened instead; iterating yields them: those of
    `edn.read_history(text, independent=True)`, so a 2-element :value is a (key, value) tuple.
    ctx: the native.Context to read on; None opens one on device 0 when the device is first needed."""

    _independent = True
    refused: str | None = None

    def flat(self, form: str = "set") -> FlatHistory:
        if form != "set":
            raise ValueError(f"a stored set history is read on the device in the set form only, not {form!r}")
        if form not in self._forms:
            from .native import EdnRefused
            try:
                self._forms[form] = self._context().read_set_edn(self.data)
            except EdnRefused as e:
                self.refused = str(e)
                self._forms[form] = flatten_ops(self.ops(), "set")
        return self._forms[form]


def _summary(history) -> dict | None:
    return history.checks() if isinstance(history, StoredLedgerHistory) else None


def _stored(data: bytes, rec) -> StoredOp:
    return StoredOp(data, rec["begin"], rec["end"])


def _flat(history, model: str) -> FlatHistory:
    if isinstance(history, FlatHistory):
        return history
    if isinstance(history, StoredLedgerHistory):
        if model in ("bank", "ledger-counters", "ledger-lookups"):
            return history.flat(model)
        return flatten_ops(history.ops(), model)
    if isinstance(history, StoredSetHistory):
        return history.flat(model) if model == "set" else flatten_ops(history.ops(), model)
    return flatten_ops(history, model)


class _Native:
    """Shares one native context per device between the checkers of a compose map."""

    def __init__(self, ctx: Context | None = None, device: int = 0, **ctx_opts) -> None:
        self._ctx = ctx
        self._device = device
        self._opts = ctx_opts

    @property
    def ctx(self) -> Context:
        if self._ctx is None:
            self._ctx = Context(device=self._device, **self._opts)
        return self._ctx


class Linearizable(Checker, _Native):
    """`(checker/linearizable {:model m})` — knossos analysis on the GPU (hot path A9).

    Result keys follow knossos: valid?, op (witness :index), previous-ok, configs (the configurations stuck at the
    witness, first 10 as jepsen.checker/linearizable keeps them, plus configs-total), configs-explored, analyzer,
    cause (when :unknown).  For keyed histories use `independent_checker(linearizable(...))`."""

    def __init__(self, model: str, ctx: Context | None = None, init_value=None, **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        if model not in _MODEL_KIND:
            raise AssertionError("The linearizable checker requires a model")  # as upstream asserts
        self.model = model
        self.init_value = init_value

    def _cmodel(self, test):
        kind = _MODEL_KIND[self.model]
        if kind == MODEL_BANK:
            accounts = list(test.get("accounts", range(1, 9)))
            return make_model(kind, accounts=accounts,
                              init_balance=test.get("initial-balances"),
                              negative_balances_ok=bool(test.get("negative-balances?", True)))
        from .history import NIL
        return make_model(kind, init_value=NIL if self.init_value is None else int(self.init_value))

    def _render_config(self, cm, c: dict) -> dict:
        from .history import NIL
        kind = _MODEL_KIND[self.model]
        if kind == MODEL_BANK:
            model = {int(cm.account_ids[i]): c["balances"][i] for i in range(cm.n_accounts)}
        elif kind == MODEL_SET:
            model = None   # the set is the union of the linearized adds
        else:
            model = None if c["state"] == NIL else c["state"]
        return {"model": model, "pending": [{"index": i} for i in c["pending"]],
                "linearized-open": [{"index": i} for i in c["linearized_open"]],
                "crashed-linearized": c["crashed_linearized"]}

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        cm = self._cmodel(test)
        r = self.ctx.check_linearizable(h, cm)
        per = []
        for k, s in enumerate(r["shards"]):
            m = {"valid?": VERDICT_NAME[s["valid"]], "analyzer": "wgl-gpu"}
            if s["valid"] == INVALID:
                m["op"] = {"index": s["witness_index"]}
                m["previous-ok"] = ({"index": s["previous_ok_index"]}
                                    if s["previous_ok_index"] >= 0 else None)
                fc = self.ctx.final_configs(h, cm, shard=k, cap=10)   # reads the table of the search just done
                m["configs"] = [self._render_config(cm, c) for c in fc["configs"]]
                m["configs-total"] = fc["total"]
            if s["valid"] == UNKNOWN:
                m["cause"] = abi.CAUSE_NAME.get(s["cause"], "unknown")
            per.append(m)
        top = {"valid?": VERDICT_NAME[r["valid"]], "configs-explored": r["configs"],
               "probes": r["probes"], "seconds-kernel": r["seconds_kernel"],
               "seconds-total": r["seconds_total"]}
        return top, per

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, self.model)
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k != "valid?"})
        return out


class SetFull(Checker, _Native):
    """`(checker/set-full {:linearizable? L})` as called at workloads/set_full.clj:157 (hot path A4)."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        checker_opts = checker_opts or {}
        self.linearizable = bool(checker_opts.get("linearizable?", False))

    @staticmethod
    def shard_maps(r: dict) -> list[dict]:
        out = []
        off = r["elem_off"]
        for s, sh in enumerate(r["shards"]):
            lo, hi = int(off[s]), int(off[s + 1])
            ids, oc = r["elem_id"][lo:hi], r["elem_outcome"][lo:hi]
            lat, dup = r["elem_latency_ms"][lo:hi], r["elem_dup_count"][lo:hi]
            stable_lat = np.sort(lat[oc == abi.SF_STABLE])
            lost_lat = np.sort(lat[oc == abi.SF_LOST])

            def quantiles(x):
                if x.size == 0:
                    return None
                # jepsen.checker/frequency-distribution: (nth sorted (min (dec n) (floor (* n p))))
                return {q: int(x[min(x.size - 1, int(np.floor(x.size * q)))]) for q in (0, 0.5, 0.95, 0.99, 1)}

            stale = [(int(i), int(l)) for i, l, o in zip(ids, lat, oc) if o == abi.SF_STABLE and l > 0]
            stale.sort(key=lambda t: -t[1])
            out.append({
                "valid?": VERDICT_NAME[sh["valid"]],
                "attempt-count": sh["attempt_count"], "stable-count": sh["stable_count"],
                "lost-count": sh["lost_count"], "lost": sorted(int(i) for i in ids[oc == abi.SF_LOST]),
                "never-read-count": sh["never_read_count"],
                "never-read": sorted(int(i) for i in ids[oc == abi.SF_NEVER_READ]),
                "stale-count": sh["stale_count"], "stale": sorted(i for i, _ in stale),
                "worst-stale": [{"element": i, "stable-latency": l} for i, l in stale[:8]],
                "stable-latencies": quantiles(stable_lat), "lost-latencies": quantiles(lost_lat),
                "duplicated-count": sh["duplicated_count"],
                "duplicated": {int(i): int(d) for i, d in zip(ids, dup) if d > 1},
            })
        return out

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_set_full(h, self.linearizable)
        return {"valid?": VERDICT_NAME[r["valid"]], "seconds-kernel": r["seconds_kernel"]}, self.shard_maps(r)

    def check(self, test, history, opts=None) -> dict:
        """Un-keyed history (what `independent/checker` hands its inner checker per key, set_full.clj:155-157)."""
        h = _flat(history, "set")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        return self.check_flat(test, h)[1][0]


class ReadAllInvokedAdds(Checker, _Native):
    """`(read-all-invoked-adds)` — workloads/set_full.clj:51-75: every :final? :ok read must contain every
    :add value invoked in its sub-history; else {:valid? false :suspect-final-reads [[index missing] ...]}.
    Evaluated on the device in the same pass as set-full (shares its read x element bit-matrix)."""

    def __init__(self, ctx: Context | None = None, **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_set_full(h, True)
        per = [{"valid?": True} for _ in range(h.n_shards)]
        for sus in r["suspect_final_reads"]:
            m = per[sus["shard"]]
            m["valid?"] = False
            m.setdefault("suspect-final-reads", []).append([sus["index"], sorted(sus["missing"])])
        return {"valid?": r["raia_valid"] == VALID}, per

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "set")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        return self.check_flat(test, h)[1][0]


class BankTotals(Checker, _Native):
    """The ledger test's `:SI` checker (tests/ledger.clj:154-192): every :ok read must sum to
    (:total-amount test); unless :negative-balances? no balance may be negative."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        self.negative_balances = bool((checker_opts or {}).get("negative-balances?", False))

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "bank")
        m = make_model(MODEL_BANK, accounts=list(test.get("accounts", range(1, 9))),
                       negative_balances_ok=self.negative_balances)
        r = self.ctx.check_bank_totals(h, m, int(test.get("total-amount", 0)))
        errors = {}
        for t, name in abi.BANK_ERR_NAME.items():
            if r["count_by_type"][t]:
                e = {"count": r["count_by_type"][t], "first": {"op": {"index": r["first_index_by_type"][t]}},
                     "worst": {"op": {"index": r["worst_index_by_type"][t]}},
                     "last": {"op": {"index": r["last_index_by_type"][t]}}}
                if name == "wrong-total":
                    e["lowest"] = {"total": r["lowest_total"], "op": {"index": r["lowest_index"]}}
                    e["highest"] = {"total": r["highest_total"], "op": {"index": r["highest_index"]}}
                errors[name] = e
        first = None
        if r["error_count"]:
            first = {"type": abi.BANK_ERR_NAME[r["first_error_type"]], "op": {"index": r["first_error_index"]}}
        out = {"valid?": r["error_count"] == 0, "read-count": r["read_count"],
               "error-count": r["error_count"], "first-error": first, "errors": errors}
        if r["reference_throws"]:
            # tests/ledger.clj:122-123: err-badness divides by (:total-amount test) = 0 (the default, :356) as soon as
            # util/max-by compares two :wrong-total errors; the reference checker throws and jepsen's check-safe
            # reports :unknown.  Same verdict here; the statistics are kept as extra keys.
            out["valid?"] = "unknown"
            out["error"] = "java.lang.ArithmeticException: Divide by zero (err-badness, tests/ledger.clj:122-123)"
        return out


class MonotonicKeys(Checker, _Native):
    """Elle's monotonic-key graph over a ledger history's :ok reads (src/tigerbeetle/elle/core.clj), on the GPU (K7).

    Every account has two counters that only grow, debits-posted and credits-posted; a read that saw a smaller
    counter than another read must come before it.  Together with real-time order (on by default) a cycle proves
    that no (real-time respecting) serial order explains the reads.  Polynomial, unaffected by crashed transfers,
    any number of accounts; weaker than `linearizable` (it does not replay transfers).  Result:
    {valid?, read-count, key-count, [cause], [op, cycle, steps]}, keys spelled [account "debits-posted"]."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        self.realtime = bool((checker_opts or {}).get("realtime?", True))

    @staticmethod
    def _key(k: int) -> list:
        return [k >> 1, COUNTER_FIELDS[k & 1]]

    def _shard_map(self, s: dict) -> dict:
        m: dict[str, Any] = {"valid?": VERDICT_NAME[s["valid"]], "read-count": s["n_reads"], "key-count": s["n_keys"]}
        if s["valid"] == UNKNOWN:
            m["cause"] = abi.CAUSE_NAME.get(s["cause"], "unknown")
        if s["valid"] == INVALID:
            w, p = {"index": s["witness_index"]}, {"index": s["partner_index"]}
            m["op"] = w
            m["cycle"] = [p, w, p]
            steps = []
            for kind, key, v, v2 in s["edges"]:
                if kind == abi.MONO_EDGE_MONOTONIC:
                    steps.append({"type": "monotonic", "key": self._key(key), "value": v, "value'": v2})
                else:   # real time: completion :index of the source, invocation :index of the target
                    steps.append({"type": "realtime", "value": v, "value'": v2})
            m["steps"] = steps
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_monotonic_keys(h, realtime=self.realtime)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"],
               "seconds-kernel": r["seconds_kernel"], "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "ledger-counters")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k not in ("valid?", "read-count")})
        return out


class CounterBounds(Checker, _Native):
    """Every counter a ledger :ok read observes held to the transfers around it, on the GPU (K8).

    debits-posted and credits-posted start at zero and only grow, so a read must hold every :ok transfer that completed
    before it was invoked (L) and nothing beyond the non-:fail transfers invoked before it completed (U).  A value below
    L is a lost transfer, above U a phantom or duplicated one.  Polynomial, any number of accounts, :info transfers only
    widen U; sound but not complete (which concurrent transfers a read saw is not decided).  Result: {valid?, read-count,
    transfer-count, error-count, [op, error]}, keys spelled [account "debits-posted"]."""

    ERROR_TYPE = {abi.CB_BELOW: "below-completed-transfers", abi.CB_ABOVE: "above-invoked-transfers"}

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)

    def _shard_map(self, s: dict) -> dict:
        m: dict[str, Any] = {"valid?": VERDICT_NAME[s["valid"]], "read-count": s["n_reads"],
                             "transfer-count": s["n_transfers"], "error-count": s["n_below"] + s["n_above"]}
        if s["valid"] == INVALID:
            m["op"] = {"index": s["witness_index"]}
            k = s["witness_key"]
            m["error"] = {"type": self.ERROR_TYPE[s["kind"]], "key": [k >> 1, COUNTER_FIELDS[k & 1]],
                          "value": s["value"], "bound": s["bound"], "transfer": {"index": s["culprit_index"]}}
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        n = h.meta.get("multi_transfer_txns", 0)
        if n:
            raise ValueError(f"{n} transfer txns have more than one [:t ...] micro-op; only the first is flattened, so "
                             "the transfers' upper bounds would be too small")
        r = self.ctx.check_counter_bounds(h)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "error-count": r["n_violations"], "seconds-kernel": r["seconds_kernel"],
               "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "ledger-counters")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k.startswith("seconds-")})
        return out


class TransferLookups(Checker, _Native):
    """The transfer records :ok lookups return held to the transfers clients issued and the counters reads show, on the
    GPU (K9).

    Reads the ledger-lookups form.  A record no transfer invoke carries (phantom), one that differs from its invocation
    (mismatch), one of a :fail transfer (failed-visible) or of a transfer invoked after the lookup completed (future),
    an id twice in one lookup (duplicate), a transfer missing from a lookup invoked after it was :ok (lost) or after an
    earlier lookup returned it (vanished), and a read's counter below the sums of a lookup completed before it or above
    those of a lookup invoked after it each prove an anomaly.  :info transfers are never required to appear.  Result:
    {valid?, lookup-count, record-count, transfer-count, read-count, error-count, errors {kind count}, [op, error]}."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)

    def _shard_map(self, s: dict) -> dict:
        errors = {abi.TL_KIND_NAME[k + 1]: n for k, n in enumerate(s["count_by_kind"]) if n}
        m: dict[str, Any] = {"valid?": VERDICT_NAME[s["valid"]], "lookup-count": s["n_lookups"],
                             "record-count": s["n_records"], "transfer-count": s["n_transfers"],
                             "read-count": s["n_reads"], "error-count": sum(errors.values()), "errors": errors}
        if s["valid"] == INVALID:
            m["op"] = {"index": s["witness_index"]}
            kind = s["kind"]
            err: dict[str, Any] = {"type": abi.TL_KIND_NAME[kind]}
            if kind >= abi.TL_READ_BELOW_LOOKUP:
                k = s["key"]
                err.update({"key": [k >> 1, COUNTER_FIELDS[k & 1]], "value": s["value"], "bound": s["bound"]})
            else:
                err["transfer-id"] = s["transfer_id"]
            if s["related_index"] >= 0:
                err["related"] = {"index": s["related_index"]}
            m["error"] = err
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_transfer_lookups(h)
        top = {"valid?": VERDICT_NAME[r["valid"]], "lookup-count": r["n_lookups"], "record-count": r["n_records"],
               "transfer-count": r["n_transfers"], "read-count": r["n_reads"], "error-count": r["n_violations"],
               "seconds-kernel": r["seconds_kernel"], "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "ledger-lookups")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k.startswith("seconds-")})
        return out


class ReadExplanations(Checker, _Native):
    """Whether one set of transfers explains every counter a ledger :ok read shows, on the GPU (K10).

    Reads the ledger-lookups form.  For each read, the transfers that must be in it (:ok, or returned by an :ok lookup,
    before it was invoked), the ones that cannot be (:fail, invoked after it completed, or absent from an :ok lookup
    invoked after it completed) and the rest, which may be; a read is explained when some subset of the last closes
    every counter it observes at once.  A read for which no single counter has such a subset is a "key" error (lost,
    phantom, duplicated or corrupt amounts), one for which each counter has one but no one subset closes all of them a
    "joint" error (torn or fractured transfers).  The search is budgeted (max-nodes, default 4096): a read it does not
    decide makes the verdict :unknown, never false.  Result: {valid?, read-count, transfer-count, explained-count,
    undecided-count, error-count, errors {kind count}, [op, error]}."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        self.max_nodes = int((checker_opts or {}).get("max-nodes", 0))

    def _shard_map(self, s: dict) -> dict:
        errors = {abi.RX_KIND_NAME[k + 1]: n for k, n in enumerate(s["count_by_kind"]) if n}
        m: dict[str, Any] = {"valid?": VERDICT_NAME[s["valid"]], "read-count": s["n_reads"],
                             "transfer-count": s["n_transfers"], "explained-count": s["n_explained"],
                             "undecided-count": s["n_undecided"], "error-count": sum(errors.values()),
                             "errors": errors}
        if s["valid"] == INVALID:
            m["op"] = {"index": s["witness_index"]}
            err: dict[str, Any] = {"type": abi.RX_KIND_NAME[s["kind"]], "must-count": s["n_must"],
                                   "may-count": s["n_may"]}
            k = s["key"]
            if k >= 0:
                err["key"] = [k >> 1, COUNTER_FIELDS[k & 1]]
            if s["kind"] == abi.RX_KEY:
                err.update({"value": s["value"], "must-sum": s["must_sum"]})
            m["error"] = err
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_read_explanations(h, self.max_nodes)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "explained-count": r["n_explained"], "undecided-count": r["n_undecided"],
               "error-count": r["n_unexplained"], "nodes": r["nodes"], "seconds-kernel": r["seconds_kernel"],
               "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "ledger-lookups")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k.startswith("seconds-") or k == "nodes"})
        return out


class ReadGaps(Checker, _Native):
    """Whether the transfers committed between two successive ledger reads explain what changed, on the GPU (K11).

    Reads the ledger-lookups form.  The :ok reads of a shard whose reads all observe every key are ordered as the
    monotonic-key check orders them (by the sum of their values, then invocation); each read closes the gap from the
    read before it (the zero state for the first).  A gap is explained when some subset of the transfers that may have
    committed inside it sums to the gap's change on every counter.  A gap with a counter going down, or whose change no
    single counter's subset produces, is a "key" error; one whose counters each close alone but not all at once a
    "joint" error; a transfer that two gaps both need is a "double" error.  Shards with a partial read are :unknown.
    The search is budgeted (max-nodes, default 4096): a gap it does not decide makes the verdict :unknown, never false.
    Result: {valid?, read-count, transfer-count, explained-count, undecided-count, error-count, errors {kind count},
    [op, lower-op, error]}."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        self.max_nodes = int((checker_opts or {}).get("max-nodes", 0))

    def _shard_map(self, s: dict) -> dict:
        errors = {abi.RG_KIND_NAME[k + 1]: n for k, n in enumerate(s["count_by_kind"]) if n}
        m: dict[str, Any] = {"valid?": VERDICT_NAME[s["valid"]], "read-count": s["n_reads"],
                             "transfer-count": s["n_transfers"], "explained-count": s["n_explained"],
                             "undecided-count": s["n_undecided"], "error-count": sum(errors.values()),
                             "errors": errors}
        if s["cause"]:
            m["cause"] = abi.CAUSE_NAME.get(s["cause"], "unknown")
        if s["valid"] == INVALID:
            m["op"] = {"index": s["witness_index"]}
            if s["lower_index"] >= 0:
                m["lower-op"] = {"index": s["lower_index"]}
            err: dict[str, Any] = {"type": abi.RG_KIND_NAME[s["kind"]], "eligible-count": s["n_eligible"]}
            k = s["key"]
            if k >= 0:
                err["key"] = [k >> 1, COUNTER_FIELDS[k & 1]]
            if s["kind"] == abi.RG_KEY:
                err["delta"] = s["delta"]
            if s["kind"] == abi.RG_DOUBLE:
                err.update({"transfer-id": s["transfer_id"], "other-op": {"index": s["other_index"]}})
            m["error"] = err
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_read_gaps(h, self.max_nodes)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "explained-count": r["n_explained"], "undecided-count": r["n_undecided"],
               "error-count": r["n_unexplained"] + r["n_double"], "nodes": r["nodes"],
               "seconds-kernel": r["seconds_kernel"], "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "ledger-lookups")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k.startswith("seconds-") or k == "nodes"})
        return out


class TransferPlacement(Checker, _Native):
    """The read-gap check with located transfers carried across gaps, on the GPU (K12).

    Reads the ledger-lookups form and orders and gaps the reads as the read-gap check does.  A transfer that one gap's
    search proves it must hold, or that only one gap of its window can still hold, is placed there and leaves every
    other gap, which is then searched again without it, round after round until nothing moves (max-rounds, default
    64).  Besides the read-gap errors ("key", "joint", "double") a transfer known to be committed before some read that
    no gap can hold is a "lost" error.  Shards with a partial read are :unknown; a gap the budget (max-nodes, default
    4096) does not decide makes the verdict :unknown, never false.
    Result: {valid?, read-count, transfer-count, explained-count, undecided-count, error-count, errors {kind count},
    placed-count, rounds, [op, lower-op, error]}."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        self.max_nodes = int((checker_opts or {}).get("max-nodes", 0))
        self.max_rounds = int((checker_opts or {}).get("max-rounds", 0))

    def _shard_map(self, s: dict) -> dict:
        errors = {abi.TP_KIND_NAME[k + 1]: n for k, n in enumerate(s["count_by_kind"]) if n}
        m: dict[str, Any] = {"valid?": VERDICT_NAME[s["valid"]], "read-count": s["n_reads"],
                             "transfer-count": s["n_transfers"], "explained-count": s["n_explained"],
                             "undecided-count": s["n_undecided"], "error-count": sum(errors.values()),
                             "errors": errors, "placed-count": s["n_placed"], "rounds": s["rounds"]}
        if s["cause"]:
            m["cause"] = abi.CAUSE_NAME.get(s["cause"], "unknown")
        if s["valid"] == INVALID:
            m["op"] = {"index": s["witness_index"]}
            if s["lower_index"] >= 0:
                m["lower-op"] = {"index": s["lower_index"]}
            err: dict[str, Any] = {"type": abi.TP_KIND_NAME[s["kind"]], "round": s["round"],
                                   "eligible-count": s["n_eligible"]}
            k = s["key"]
            if k >= 0:
                err["key"] = [k >> 1, COUNTER_FIELDS[k & 1]]
            if s["kind"] == abi.TP_KEY:
                err["delta"] = s["delta"]
            if s["kind"] in (abi.TP_DOUBLE, abi.TP_LOST):
                err.update({"transfer-id": s["transfer_id"], "other-op": {"index": s["other_index"]}})
            m["error"] = err
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_transfer_placement(h, self.max_nodes, self.max_rounds)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "explained-count": r["n_explained"], "undecided-count": r["n_undecided"],
               "error-count": r["n_unexplained"] + r["n_double"] + r["n_lost"], "placed-count": r["n_placed"],
               "rounds": r["rounds"], "nodes": r["nodes"], "seconds-kernel": r["seconds_kernel"],
               "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "ledger-lookups")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k.startswith("seconds-") or k == "nodes"})
        return out


class SerialWitness(Checker, _Native):
    """A proof that a ledger history is linearizable, on the GPU (K13), or nothing.

    Reads the ledger-lookups form and runs the transfer-placement check (max-nodes, max-rounds).  For a shard it calls
    valid, one explanation is chosen per read gap, no transfer in two (max-rounds witness rounds), and the serial order
    they give (each read after the transfers of the gaps up to it) is checked against real time.  A shard that passes
    is :valid? true: its reads and transfers are linearizable for the per-account counters, and so for the bank model
    with negative balances allowed (the ledger test's :linear question); lookups are not placed.  Otherwise it is
    :unknown with a cause ("partial-read", "anomaly", "undecided", "no-witness", "real-time"); never false, since the
    anomalies are the other ledger checks' business.
    Result: {valid?, read-count, transfer-count, committed-count, committed-crashed-count, after-count, rounds, [cause,
    op, transfer-id]}."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        _Native.__init__(self, ctx, **ctx_opts)
        self.max_nodes = int((checker_opts or {}).get("max-nodes", 0))
        self.max_rounds = int((checker_opts or {}).get("max-rounds", 0))

    def _shard_map(self, s: dict) -> dict:
        m: dict[str, Any] = {"valid?": VERDICT_NAME[s["valid"]], "read-count": s["n_reads"],
                             "transfer-count": s["n_transfers"], "committed-count": s["n_committed"],
                             "committed-crashed-count": s["n_committed_crashed"], "after-count": s["n_after"],
                             "rounds": s["rounds"]}
        if s["cause"]:
            m["cause"] = abi.CAUSE_NAME.get(s["cause"], "unknown")
        if s["fail_index"] >= 0:
            m["op"] = {"index": s["fail_index"]}
        if s["transfer_id"] >= 0:
            m["transfer-id"] = s["transfer_id"]
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_serial_witness(h, self.max_nodes, self.max_rounds)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "committed-count": r["n_committed"], "committed-crashed-count": r["n_committed_crashed"],
               "after-count": r["n_after"], "rounds": r["rounds"], "nodes": r["nodes"],
               "seconds-kernel": r["seconds_kernel"], "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, "ledger-lookups")
        if h.n_shards != 1:
            raise ValueError("history has independent keys: wrap with independent_checker(...)")
        top, per = self.check_flat(test, h)
        out = dict(per[0])
        out.update({k: v for k, v in top.items() if k.startswith("seconds-") or k == "nodes"})
        return out


class RepairedWitness(SerialWitness):
    """The serial-witness check with repairs, on the GPU (K14): a shard the serial-witness check leaves :unknown
    ("no-witness" or "real-time") gets up to max-repairs repair rounds, each banning the (transfer, gap) pairs the
    failure blames and choosing the released gaps' explanations again; a VALID is the same proof, and a shard the
    serial-witness check proves comes back unchanged.  Result: SerialWitness's map plus repairs and ban-count."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        SerialWitness.__init__(self, checker_opts, ctx, **ctx_opts)
        self.max_repairs = int((checker_opts or {}).get("max-repairs", 0))

    def _shard_map(self, s: dict) -> dict:
        m = SerialWitness._shard_map(self, s)
        m.update({"repairs": s["repairs"], "ban-count": s["n_bans"]})
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_repaired_witness(h, self.max_nodes, self.max_rounds, self.max_repairs)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "committed-count": r["n_committed"], "committed-crashed-count": r["n_committed_crashed"],
               "after-count": r["n_after"], "rounds": r["rounds"], "repairs": r["repairs"],
               "ban-count": r["n_bans"], "nodes": r["nodes"], "seconds-kernel": r["seconds_kernel"],
               "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]


class LiftedWitness(RepairedWitness):
    """The repaired serial witness with lifted bans, on the GPU (K15): a shard whose repairs stop because a repair
    recorded no new ban gets up to max-lifts lift steps, each letting the failing gaps take back transfers their own
    bans held (once per pair) before the repairs resume; a VALID is the same proof, and a shard the repaired witness
    proves comes back unchanged.  Result: RepairedWitness's map plus lifts and lifted-count."""

    def __init__(self, checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                 **ctx_opts) -> None:
        RepairedWitness.__init__(self, checker_opts, ctx, **ctx_opts)
        self.max_lifts = int((checker_opts or {}).get("max-lifts", 0))

    def _shard_map(self, s: dict) -> dict:
        m = RepairedWitness._shard_map(self, s)
        m.update({"lifts": s["lifts"], "lifted-count": s["n_lifted"]})
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_lifted_witness(h, self.max_nodes, self.max_rounds, self.max_repairs, self.max_lifts)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "committed-count": r["n_committed"], "committed-crashed-count": r["n_committed_crashed"],
               "after-count": r["n_after"], "rounds": r["rounds"], "repairs": r["repairs"],
               "ban-count": r["n_bans"], "lifts": r["lifts"], "lifted-count": r["n_lifted"], "nodes": r["nodes"],
               "seconds-kernel": r["seconds_kernel"], "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]


class ClassWitness(LiftedWitness):
    """The lifted serial witness, then a class pass on the GPU (K16) on every shard it leaves unknown (undecided,
    no-witness or real-time): starting again from the transfer-placement check's owners, the witness rounds treat
    crashed transfers with the same debit, credit, amount and lookup bounds as one class, gather at most as many of a
    class as the gap can use, and hand each gap the earliest members of the class; the same real-time pass and re-sum
    make a :valid? true the same proof.  A shard the lifted witness proves comes back unchanged.  Result:
    LiftedWitness's map plus class-rounds and handed-count, and class-cause when the class pass ran and failed."""

    def _shard_map(self, s: dict) -> dict:
        m = LiftedWitness._shard_map(self, s)
        m.update({"class-rounds": s["class_rounds"], "handed-count": s["n_handed"]})
        if s["class_cause"]:
            m["class-cause"] = abi.CAUSE_NAME[s["class_cause"]]
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_class_witness(h, self.max_nodes, self.max_rounds, self.max_repairs, self.max_lifts)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "committed-count": r["n_committed"], "committed-crashed-count": r["n_committed_crashed"],
               "after-count": r["n_after"], "rounds": r["rounds"], "repairs": r["repairs"],
               "ban-count": r["n_bans"], "lifts": r["lifts"], "lifted-count": r["n_lifted"],
               "class-rounds": r["class_rounds"], "handed-count": r["n_handed"], "nodes": r["nodes"],
               "seconds-kernel": r["seconds_kernel"], "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]


class LookupWitness(ClassWitness):
    """The class witness, then every :ok lookup placed in the serial order it proves, on the GPU (K17): each lookup
    goes where it returns exactly the transfers committed before it, the lookups of one read gap must return nested
    sets, and one real-time pass checks the reads, transfers and lookups together.  A :valid? true then covers the
    whole ledger history, lookups included.  A shard whose lookups have no place is :unknown with cause "lookup" and
    lookup-op, the lookup that failed.  Result: ClassWitness's map plus lookups-placed-count, and lookup-cause."""

    def _shard_map(self, s: dict) -> dict:
        m = ClassWitness._shard_map(self, s)
        m["lookups-placed-count"] = s["n_lookups_placed"]
        if s["lookup_cause"]:
            m["lookup-cause"] = abi.CAUSE_NAME[s["lookup_cause"]]
            m["lookup-op"] = {"index": s["lookup_fail_index"]}
        return m

    def check_flat(self, test, h: FlatHistory) -> tuple[dict, list[dict]]:
        r = self.ctx.check_lookup_witness(h, self.max_nodes, self.max_rounds, self.max_repairs, self.max_lifts)
        top = {"valid?": VERDICT_NAME[r["valid"]], "read-count": r["n_reads"], "transfer-count": r["n_transfers"],
               "committed-count": r["n_committed"], "committed-crashed-count": r["n_committed_crashed"],
               "after-count": r["n_after"], "rounds": r["rounds"], "repairs": r["repairs"],
               "ban-count": r["n_bans"], "lifts": r["lifts"], "lifted-count": r["n_lifted"],
               "class-rounds": r["class_rounds"], "handed-count": r["n_handed"],
               "lookups-placed-count": r["n_lookups_placed"], "nodes": r["nodes"],
               "seconds-kernel": r["seconds_kernel"], "seconds-total": r["seconds_total"]}
        return top, [self._shard_map(s) for s in r["shards"]]


class Compose(Checker):
    """`(checker/compose {name checker ...})`: run each, `:valid?` = merge-valid of the results."""

    def __init__(self, checkers: Mapping[str, Checker]) -> None:
        self.checkers = dict(checkers)

    def check(self, test, history, opts=None) -> dict:
        out = {k: check_safe(c, test, history, opts) for k, c in self.checkers.items()}
        out["valid?"] = merge_valid_values(r["valid?"] for r in list(out.values()))
        return out


class Independent(Checker):
    """`(independent/checker inner)`: split the history by key, check every sub-history, merge
    (SURVEY A.2).  Unlike the JVM original the split is the CSR partition of the flattened history
    and keyed-aware inner checkers (Linearizable, SetFull, Compose of those) receive ALL shards in one
    native call, so the GPU owns the fan-out."""

    def __init__(self, inner: Checker, model: str | None = None) -> None:
        self.inner = inner
        self.model = model

    def _model(self) -> str:
        if self.model:
            return self.model
        c = self.inner
        if isinstance(c, Compose):
            c = next(iter(c.checkers.values()))
        if isinstance(c, Linearizable):
            return c.model
        if isinstance(c, (MonotonicKeys, CounterBounds)):
            return "ledger-counters"
        if isinstance(c, (TransferLookups, ReadExplanations, ReadGaps, TransferPlacement, SerialWitness)):
            return "ledger-lookups"
        return "set"

    def _per_key(self, checker: Checker, test, h: FlatHistory, opts) -> list[dict]:
        if isinstance(checker, (Linearizable, SetFull, ReadAllInvokedAdds, MonotonicKeys, CounterBounds,
                                TransferLookups, ReadExplanations, ReadGaps, TransferPlacement, SerialWitness)):
            try:
                return checker.check_flat(test, h)[1]
            except Exception:  # noqa: BLE001
                err = traceback.format_exc()
                return [{"valid?": "unknown", "error": err} for _ in range(h.n_shards)]
        if isinstance(checker, Compose):
            cols = {name: self._per_key(c, test, h, opts) for name, c in checker.checkers.items()}
            out = []
            for s in range(h.n_shards):
                m = {name: col[s] for name, col in cols.items()}
                m["valid?"] = merge_valid_values(r["valid?"] for r in list(m.values()))
                out.append(m)
            return out
        # generic checker: one call per sub-history
        return [check_safe(checker, test, h.shard(s),
                           dict(opts or {}, **{"history-key": int(h.key_ids[s])}))
                for s in range(h.n_shards)]

    def check(self, test, history, opts=None) -> dict:
        h = _flat(history, self._model())
        per = self._per_key(self.inner, test, h, opts)
        results = {int(k): r for k, r in zip(h.key_ids, per)}
        failures = [k for k, r in results.items() if r["valid?"] is not True]
        return {"valid?": merge_valid_values(r["valid?"] for r in per) if per else True,
                "results": results, "failures": failures}


# ---- constructors with the reference's names ---------------------------------------------------------
def linearizable(opts: Mapping[str, Any], **kw) -> Linearizable:
    """`(checker/linearizable {:model :cas-register})`"""
    return Linearizable(opts["model"], init_value=opts.get("init-value"), **kw)


def set_full(opts: Mapping[str, Any] | None = None, **kw) -> SetFull:
    """`(checker/set-full {:linearizable? true})` — set_full.clj:157"""
    return SetFull(opts, **kw)


def read_all_invoked_adds(**kw) -> ReadAllInvokedAdds:
    """`(read-all-invoked-adds)` — set_full.clj:51-75, :158"""
    return ReadAllInvokedAdds(**kw)


def bank_checker(opts: Mapping[str, Any] | None = None, **kw) -> BankTotals:
    """`(ledger/checker {:negative-balances? true})` — tests/ledger.clj:154-192, :363"""
    return BankTotals(opts, **kw)


def monotonic_key_checker(opts: Mapping[str, Any] | None = None, **kw) -> MonotonicKeys:
    """Elle's monotonic-key check over the ledger counters; {"realtime?": False} gives the literal elle/core.clj
    graph without real-time edges."""
    return MonotonicKeys(opts, **kw)


def counter_bounds_checker(opts: Mapping[str, Any] | None = None, **kw) -> CounterBounds:
    """Every ledger read's counters against the bounds the :ok and :info transfers around it put on them (K8)."""
    return CounterBounds(opts, **kw)


def transfer_lookup_checker(opts: Mapping[str, Any] | None = None, **kw) -> TransferLookups:
    """The looked-up transfer records against the transfers clients issued and the counters reads show (K9)."""
    return TransferLookups(opts, **kw)


def read_explanation_checker(opts: Mapping[str, Any] | None = None, **kw) -> ReadExplanations:
    """Whether one set of transfers explains every counter each ledger read shows (K10); {"max-nodes": n} sets the
    per-read search budget."""
    return ReadExplanations(opts, **kw)


def read_gap_checker(opts: Mapping[str, Any] | None = None, **kw) -> ReadGaps:
    """Whether the transfers committed between two successive ledger reads explain what changed (K11);
    {"max-nodes": n} sets the per-gap search budget."""
    return ReadGaps(opts, **kw)


def transfer_placement_checker(opts: Mapping[str, Any] | None = None, **kw) -> TransferPlacement:
    """The read-gap check with located transfers carried across gaps to a fixpoint (K12); {"max-nodes": n} sets the
    per-gap search budget and {"max-rounds": n} the number of rounds."""
    return TransferPlacement(opts, **kw)


def serial_witness_checker(opts: Mapping[str, Any] | None = None, **kw) -> SerialWitness:
    """A proof of linearizability for ledger histories, or :unknown (K13); {"max-nodes": n} and {"max-rounds": n} as
    for the transfer-placement check it runs first."""
    return SerialWitness(opts, **kw)


def repaired_witness_checker(opts: Mapping[str, Any] | None = None, **kw) -> RepairedWitness:
    """The serial-witness check with repair rounds (K14); {"max-nodes": n} and {"max-rounds": n} as for the
    serial-witness check, {"max-repairs": n} the repair rounds (default abi.RW_DEFAULT_MAX_REPAIRS)."""
    return RepairedWitness(opts, **kw)


def lifted_witness_checker(opts: Mapping[str, Any] | None = None, **kw) -> LiftedWitness:
    """The repaired serial witness with lift steps (K15); {"max-nodes" "max-rounds" "max-repairs"} as for the
    repaired serial witness, {"max-lifts": n} the lift steps (default abi.LW_DEFAULT_MAX_LIFTS)."""
    return LiftedWitness(opts, **kw)


def class_witness_checker(opts: Mapping[str, Any] | None = None, **kw) -> ClassWitness:
    """The lifted serial witness with a class pass (K16); {"max-nodes" "max-rounds" "max-repairs" "max-lifts"} as for
    the lifted serial witness ("max-rounds" also bounds the class rounds)."""
    return ClassWitness(opts, **kw)


def lookup_witness_checker(opts: Mapping[str, Any] | None = None, **kw) -> LookupWitness:
    """The class witness with its lookups placed (K17); {"max-nodes" "max-rounds" "max-repairs" "max-lifts"} as for
    the class witness."""
    return LookupWitness(opts, **kw)


def compose(checkers: Mapping[str, Checker]) -> Compose:
    return Compose(checkers)


def independent_checker(inner: Checker, model: str | None = None) -> Independent:
    return Independent(inner, model)


# =====================================================================================================
# The ledger test's remaining (host-side, O(events)) checkers — SURVEY §8(f) N3.  In the reference these
# are plain Clojure seq operations over the op maps with no arithmetic worth a kernel; they are restated
# here on the host so that the whole `compose` map of tests/ledger.clj:363-367 can be served by this
# package.  They consume op maps (not the flattened arrays: they need the :l-t ops and :final? flags).
# =====================================================================================================
def _is_client(op) -> bool:
    p = op.get("process", op.get(":process"))
    return isinstance(p, (int, np.integer)) and not isinstance(p, bool)


def _g(op, name, default=None):
    return op.get(name, op.get(":" + name, default))


def _kw(x):
    return x[1:] if isinstance(x, str) and x.startswith(":") else x


def _txn_f(op):
    """tests/ledger.clj:17-21 op->txn-f: the first micro-op's tag."""
    v = _g(op, "value")
    if not v:
        return None
    first = v[0] if isinstance(v, (list, tuple)) else None
    return _kw(first[0]) if first else None


def _freeze(x):
    if isinstance(x, dict):
        return tuple(sorted((k, _freeze(v)) for k, v in x.items()))
    if isinstance(x, (list, tuple)):
        return tuple(_freeze(v) for v in x)
    if isinstance(x, (set, frozenset)):
        return frozenset(_freeze(v) for v in x)
    return x


class UnexpectedOps(Checker):
    """`(unexpected-ops)` — tests/ledger.clj:194-220: never-resolved invokes and :fail ops mark the
    result :unknown ({:valid? :unknown :open-ops [...] :fail-ops [...]})."""

    def check(self, test, history, opts=None) -> dict:
        s = _summary(history)
        if s is not None:
            return self.from_summary(s, history.data)
        hist = [op for op in history if _is_client(op)]
        end_time = _g(hist[-1], "time", 0) if hist else 0
        open_by_process: dict = {}
        for op in hist:  # knossos.history/unmatched-invokes
            t = _kw(_g(op, "type"))
            p = _g(op, "process")
            if t == "invoke":
                open_by_process[p] = op
            else:
                open_by_process.pop(p, None)
        open_ops = sorted(open_by_process.values(), key=lambda o: _g(o, "index", 0))
        opens = [[(end_time - _g(o, "time", 0)) / 1e6, o] for o in open_ops][::-1]  # util/nanos->ms, rseq
        fails = [op for op in hist if _kw(_g(op, "type")) == "fail"]
        out: dict = {"valid?": True}
        if opens:
            out.update({"valid?": "unknown", "open-ops": opens})
        if fails:
            out.update({"valid?": "unknown", "fail-ops": fails})
        return out

    @staticmethod
    def from_summary(s: Mapping[str, Any], data: bytes) -> dict:
        """The result from a stored history's device summary (`Context.ledger_edn_checks`) and its bytes; an absent
        :time or :index is 0 in the records, as `_g` reads it."""
        end_time = int(s["last"]["time"]) if s["last"] is not None else 0
        open_recs = sorted(s["open"], key=lambda r: int(r["first"]))   # the order processes enter open_by_process
        open_recs = sorted(open_recs, key=lambda r: int(r["index"]))
        opens = [[(end_time - int(r["time"])) / 1e6, _stored(data, r)] for r in open_recs][::-1]
        fails = [_stored(data, r) for r in s["fails"]]
        out: dict = {"valid?": True}
        if opens:
            out.update({"valid?": "unknown", "open-ops": opens})
        if fails:
            out.update({"valid?": "unknown", "fail-ops": fails})
        return out


class LookupAllInvokedTransfers(Checker):
    """`(lookup-all-invoked-transfers)` — tests/ledger.clj:222-252: every :final? :ok :l-t lookup must
    contain the id of every invoked transfer."""

    def check(self, test, history, opts=None) -> dict:
        s = _summary(history)
        if s is not None:
            return self.from_summary(s, history.data)
        hist = [op for op in history if _is_client(op)]
        invoked = set()
        for op in hist:
            if _txn_f(op) == "t" and _kw(_g(op, "type")) == "invoke":
                for micro in _g(op, "value"):
                    invoked.add(micro[1])
        suspects = []
        for op in hist:
            if _txn_f(op) == "l-t" and _kw(_g(op, "type")) == "ok" and _g(op, "final?"):
                ids = {micro[1] for micro in _g(op, "value")}
                if invoked - ids:
                    suspects.append(op)
        out: dict = {"valid?": True}
        if suspects:
            out.update({"valid?": False, "suspect-final-lookups": suspects})
        return out

    @staticmethod
    def from_summary(s: Mapping[str, Any], data: bytes) -> dict:
        suspects = [_stored(data, r) for r in s["final_lookups"] if r["suspect"]]
        out: dict = {"valid?": True}
        if suspects:
            out.update({"valid?": False, "suspect-final-lookups": suspects})
        return out


class FinalReads(Checker):
    """`(final-reads)` — tests/ledger.clj:254-282: final reads (and final :l-t lookups) must exist and be
    all equal: exactly one distinct :value among the :final? :ok :r ops, and among the :l-t ones."""

    def check(self, test, history, opts=None) -> dict:
        s = _summary(history)
        if s is not None:
            return self.from_summary(s, history.data)
        hist = [op for op in history if _is_client(op)]

        def finals(tag):
            return {_freeze(_g(op, "value")) for op in hist
                    if _txn_f(op) == tag and _kw(_g(op, "type")) == "ok" and _g(op, "final?")}

        reads, lookups = finals("r"), finals("l-t")
        out: dict = {"valid?": True}
        if len(reads) != 1:
            out.update({"valid?": False, "unequal-final-reads": reads})
        if len(lookups) != 1:
            out.update({"valid?": False, "unequal-final-lookups": lookups})
        return out

    @staticmethod
    def from_summary(s: Mapping[str, Any], data: bytes) -> dict:
        """Only when a kind does not have exactly one class are its values needed: one op per class is parsed."""
        def finals(recs, n_classes):
            first: dict = {}
            for r in recs:
                first.setdefault(int(r["cls"]), r)
            values = {_freeze(_g(_stored(data, r), "value")) for r in first.values()}
            assert len(values) == n_classes, (len(values), n_classes)
            return values

        out: dict = {"valid?": True}
        if s["n_read_classes"] != 1:
            out.update({"valid?": False, "unequal-final-reads": finals(s["final_reads"], s["n_read_classes"])})
        if s["n_lookup_classes"] != 1:
            out.update({"valid?": False,
                        "unequal-final-lookups": finals(s["final_lookups"], s["n_lookup_classes"])})
        return out


class Stats(Checker):
    """`(checker/stats)` as composed at core.clj:144 [UPSTREAM-RECALL, jepsen.checker/stats]: success / failure counts of
    the client completions, overall and by :f; valid only when every :f has at least one :ok completion
    ({:valid? false} otherwise: an operation that never once succeeded makes the rest of the analysis vacuous).
    Host code, as in the reference (a linear pass over the history; nothing to put on a GPU)."""

    @staticmethod
    def _counts(ok: int, fail: int, info: int) -> dict:
        return {"valid?": ok > 0, "count": ok + fail + info, "ok-count": ok, "fail-count": fail, "info-count": info}

    @staticmethod
    def _tally(ops) -> dict:
        ok = sum(1 for o in ops if _kw(_g(o, "type")) == "ok")
        fail = sum(1 for o in ops if _kw(_g(o, "type")) == "fail")
        info = sum(1 for o in ops if _kw(_g(o, "type")) == "info")
        return Stats._counts(ok, fail, info)

    def check(self, test, history, opts=None) -> dict:
        s = _summary(history)
        if s is not None:
            return self.from_summary(s)
        done = [op for op in history if _is_client(op) and _kw(_g(op, "type")) != "invoke"]
        by_f: dict = {}
        for op in done:
            by_f.setdefault(_kw(_g(op, "f")), []).append(op)
        out = self._tally(done)
        out["by-f"] = {f: self._tally(ops) for f, ops in sorted(by_f.items(), key=lambda kv: str(kv[0]))}
        out["valid?"] = merge_valid_bool([r["valid?"] for r in out["by-f"].values()])
        return out

    @staticmethod
    def from_summary(s: Mapping[str, Any]) -> dict:
        """Every client op of a stored ledger history is :f :txn (the device refuses others)."""
        out = Stats._counts(s["n_ok"], s["n_fail"], s["n_info"])
        out["by-f"] = {"txn": Stats._counts(s["n_ok"], s["n_fail"], s["n_info"])} if out["count"] else {}
        out["valid?"] = merge_valid_bool([r["valid?"] for r in out["by-f"].values()])
        return out


def merge_valid_bool(vs) -> Any:
    """jepsen.checker/merge-valid over {True, "unknown", False} values (True for an empty collection)."""
    order = {True: 0, "unknown": 1, False: 2}
    worst = True
    for v in vs:
        if order[v] > order[worst]:
            worst = v
    return worst


def stats() -> Stats:
    return Stats()


def unexpected_ops() -> UnexpectedOps:
    return UnexpectedOps()


def lookup_all_invoked_transfers() -> LookupAllInvokedTransfers:
    return LookupAllInvokedTransfers()


def final_reads() -> FinalReads:
    return FinalReads()


def ledger_checker(checker_opts: Mapping[str, Any] | None = None, ctx: Context | None = None,
                   linear: bool = True, monotonic: bool = False, counter_bounds: bool = False,
                   transfer_lookups: bool = False, read_explanations: bool = False,
                   read_gaps: bool = False, transfer_placement: bool = False,
                   serial_witness: bool = False, repaired_witness: bool = False,
                   lifted_witness: bool = False, class_witness: bool = False,
                   lookup_witness: bool = False) -> Compose:
    """The ledger test's checker (tests/ledger.clj:363-367) minus the gnuplot plotter, plus the
    linearizability search the north-star adds and, with monotonic=True, the monotonic-key check, with
    counter_bounds=True, the counter-bounds check, with transfer_lookups=True, the transfer-lookup check, with
    read_explanations=True, the read-explanation check, with read_gaps=True, the read-gap check, with
    transfer_placement=True, the transfer-placement check, with serial_witness=True, the serial-witness check, with
    repaired_witness=True, the repaired serial witness, with lifted_witness=True, the lifted serial witness, with
    class_witness=True, the class witness and, with lookup_witness=True, the lookup witness:
        {:SI (checker opts) :lookup-transfers ... :final-reads ... :unexpected-ops ... [:linear ...] [:monotonic ...]
         [:counter-bounds ...] [:transfer-lookups ...] [:read-explanations ...] [:read-gaps ...]
         [:transfer-placement ...] [:serial-witness ...] [:repaired-witness ...] [:lifted-witness ...]
         [:class-witness ...] [:lookup-witness ...]}"""
    cs: dict[str, Checker] = {"SI": bank_checker(checker_opts, ctx=ctx),
                              "lookup-transfers": lookup_all_invoked_transfers(),
                              "final-reads": final_reads(), "unexpected-ops": unexpected_ops()}
    if linear:
        cs["linear"] = linearizable({"model": "bank"}, ctx=ctx)
    if monotonic:
        cs["monotonic"] = monotonic_key_checker(ctx=ctx)
    if counter_bounds:
        cs["counter-bounds"] = counter_bounds_checker(ctx=ctx)
    if transfer_lookups:
        cs["transfer-lookups"] = transfer_lookup_checker(ctx=ctx)
    if read_explanations:
        cs["read-explanations"] = read_explanation_checker(ctx=ctx)
    if read_gaps:
        cs["read-gaps"] = read_gap_checker(ctx=ctx)
    if transfer_placement:
        cs["transfer-placement"] = transfer_placement_checker(ctx=ctx)
    if serial_witness:
        cs["serial-witness"] = serial_witness_checker(ctx=ctx)
    if repaired_witness:
        cs["repaired-witness"] = repaired_witness_checker(ctx=ctx)
    if lifted_witness:
        cs["lifted-witness"] = lifted_witness_checker(ctx=ctx)
    if class_witness:
        cs["class-witness"] = class_witness_checker(ctx=ctx)
    if lookup_witness:
        cs["lookup-witness"] = lookup_witness_checker(ctx=ctx)
    return compose(cs)


def set_full_workload_checker(ctx: Context | None = None) -> Independent:
    """The set-full workload's checker (workloads/set_full.clj:155-158) on one context:
        (independent/checker (checker/compose {:set-full (checker/set-full {:linearizable? true})
                                               :read-all-invoked-adds (read-all-invoked-adds)}))
    It is the set-full counterpart of `ledger_checker()`; given a `StoredSetHistory`, it reads the file on the device.
    ctx: the context both checkers run on; None opens one on device 0 now."""
    if ctx is None:
        ctx = Context(device=0)
    return independent_checker(compose({"set-full": set_full({"linearizable?": True}, ctx=ctx),
                                        "read-all-invoked-adds": read_all_invoked_adds(ctx=ctx)}))
