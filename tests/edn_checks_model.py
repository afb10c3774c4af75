"""A Python model of K19's summary (`Context.ledger_edn_checks`): the same dict, computed from the bytes of a small
history.edn with edn.loads and the rules of the issue's four checkers, for the CPU tier (it feeds the host assembly
`from_summary`) and as a second reference for the device's counts, ordinals, suspect bits and classes."""
import numpy as np

from jepsen_tigerbeetle_b200 import abi, edn
from jepsen_tigerbeetle_b200.checker import _freeze


def op_spans(data: bytes) -> list:
    """[begin, end) of every op map: the maps at depth 0, or inside the one top-level vector.  Strings are skipped;
    comments are not supported (the device refuses them)."""
    opens, spans, stack, top = {"[": "]", "{": "}", "(": ")"}, [], [], []
    i, n = 0, len(data)
    while i < n:
        c = chr(data[i])
        if c == '"':
            i += 1
            while data[i] != ord('"'):
                i += 2 if data[i] == ord("\\") else 1
        elif c in opens:
            if not stack:
                top.append(c)
            stack.append(i)
        elif c in ")]}":
            b = stack.pop()
            spans.append((len(stack), b, i + 1))
        i += 1
    base = 1 if len(top) == 1 and top[0] in "[(" else 0
    return sorted((b, e) for d, b, e in spans if d == base and chr(data[b]) == "{")


def _flag(k, op, begin, end, **kw):
    r = np.zeros(1, abi.EDN_FLAG_DTYPE)[0]
    r["op"], r["begin"], r["end"], r["first"], r["cls"] = k, begin, end, -1, -1
    r["has_time"], r["has_index"] = "time" in op, "index" in op
    r["time"], r["index"] = op.get("time", 0), op.get("index", 0)
    for key, v in kw.items():
        r[key] = v
    return r


def _arr(recs):
    return np.array(recs, dtype=abi.EDN_FLAG_DTYPE) if recs else np.zeros(0, abi.EDN_FLAG_DTYPE)


def summarize(data: bytes) -> dict:
    spans = op_spans(data)
    ops = [edn.loads(data[b:e].decode()) for b, e in spans]
    client = [k for k, op in enumerate(ops)
              if isinstance(op.get("process"), int) and not isinstance(op.get("process"), bool)]

    def tag(op):
        v = op.get("value")
        return v[0][0] if isinstance(v, list) and v else None

    def final(op, t):
        return tag(op) == t and op["type"] == "ok" and op.get("final?")

    s = {name: 0 for name in abi.EDN_CHECKS_COUNTS}
    s.update(refused=None, n_ops=len(ops), n_client=len(client))
    for t in ("ok", "fail", "info"):
        s["n_" + t] = sum(ops[k]["type"] == t for k in client)
    rec = lambda k, **kw: _flag(k, ops[k], *spans[k], **kw)   # noqa: E731
    s["last"] = rec(client[-1]) if client else None
    by_process: dict = {}
    for k in client:
        by_process.setdefault(ops[k]["process"], []).append(k)
    open_recs = []
    for p in sorted(by_process):
        ks = by_process[p]
        if ops[ks[-1]]["type"] == "invoke":
            j = len(ks) - 1
            while j > 0 and ops[ks[j - 1]]["type"] == "invoke":
                j -= 1
            open_recs.append(rec(ks[-1], first=ks[j]))
    s["open"] = _arr(open_recs)
    s["fails"] = _arr([rec(k) for k in client if ops[k]["type"] == "fail"])
    invoked = {m[1] for k in client if tag(ops[k]) == "t" and ops[k]["type"] == "invoke" for m in ops[k]["value"]}
    s["n_invoked"] = len(invoked)
    for kind, t in (("reads", "r"), ("lookups", "l-t")):
        classes: dict = {}
        recs = []
        for k in client:
            if final(ops[k], t):
                cls = classes.setdefault(_freeze(ops[k]["value"]), len(classes))
                sus = t == "l-t" and bool(invoked - {m[1] for m in ops[k]["value"]})
                recs.append(rec(k, cls=cls, suspect=sus))
        s["final_" + kind] = _arr(recs)
        s["n_final_" + kind] = len(recs)
        s["n_%s_classes" % kind[:-1]] = len(classes)
    s["n_open"], s["n_fail"] = len(open_recs), len(s["fails"])
    s["n_suspect"] = int(s["final_lookups"]["suspect"].sum()) if len(s["final_lookups"]) else 0
    return s


# ---- hand cases: each a history.edn the four checkers and the device summary are compared on ----------------------
def _t(i, d=1, c=2, a=3):
    return ["t", i, {"debit-acct": d, "credit-acct": c, "amount": a}]


def _lt(i, d=1, c=2, a=3):
    return ["l-t", i, {"debit-acct": d, "credit-acct": c, "amount": a}]


def _r(acct, d=0, c=0):
    return ["r", acct, {"debits-posted": d, "credits-posted": c}]


def _op(type_, process, value, index=None, time=None, final=False):
    op = {"type": type_, "process": process, "f": "txn", "value": value}
    if index is not None:
        op["index"] = index
    if time is not None:
        op["time"] = time
    if final:
        op["final?"] = True
    return op


def _edn(ops) -> bytes:
    from jepsen_tigerbeetle_b200 import stored
    return stored.write_edn(ops)


def _transfers_then_finals(final_lookups, final_reads=()):
    """Three transfers (one multi-transfer txn with ids 2 and 3), then the given final lookups and reads."""
    ops = [_op("invoke", 0, [_t(1)], 0, 10), _op("ok", 0, [_t(1)], 1, 20),
           _op("invoke", 1, [_t(2), _t(3, 2, 1)], 2, 30), _op("ok", 1, [_t(2), _t(3, 2, 1)], 3, 40)]
    k = 4
    for v in final_reads:
        ops += [_op("invoke", 2, [["r", 1, None]], k, 10 * k, True), _op("ok", 2, v, k + 1, 10 * k + 5, True)]
        k += 2
    for v in final_lookups:
        ops += [_op("invoke", 3, [["l-t", 1, None]], k, 10 * k, True), _op("ok", 3, v, k + 1, 10 * k + 5, True)]
        k += 2
    return _edn(ops)


ALL = [_lt(1), _lt(2), _lt(3, 2, 1)]
READ = [_r(1, 3, 0), _r(2, 0, 3)]
HAND_CASES = {
    "open invokes": _edn([
        _op("invoke", 0, [_t(1)], 0, 10), _op("invoke", 1, [_t(2)], 1, 11), _op("ok", 1, [_t(2)], 2, 12),
        _op("invoke", 1, [_t(3)], 3, 13), _op("invoke", 2, [["r", 1, None]], 4, 14),
        _op("invoke", 2, [["r", 1, None]], 5, 15), _op("invoke", 3, [_t(4)], None, 16),
        {"type": "info", "process": "nemesis", "f": "kill", "value": None, "time": 17},
        _op("invoke", 4, [_t(5)], 7, None)]),
    "open invokes with equal indices": _edn([
        _op("invoke", 5, [_t(1)], None, 1), _op("invoke", 2, [_t(2)], None, 2), _op("invoke", 7, [_t(3)], 0, 3),
        _op("ok", 5, [_t(1)], None, 4), _op("invoke", 5, [_t(4)], None, 5)]),
    "fail and info": _edn([
        _op("invoke", 0, [_t(1)], 0, 10), _op("fail", 0, [_t(1)], 1, 20), _op("invoke", 1, [_t(2)], 2, 30),
        _op("info", 1, [_t(2)], 3, 40), _op("invoke", 2, [["r", 1, None]], 4, 50),
        _op("ok", 2, [_r(1, 3, 0)], 5, 60), _op("invoke", 0, [_t(3)], 6, 70), _op("fail", 0, [_t(3)], 7, 80)]),
    "valid finals": _transfers_then_finals([ALL, ALL], [READ, READ]),
    "a final lookup missing one id": _transfers_then_finals([ALL, [_lt(1), _lt(3, 2, 1)]], [READ]),
    "missing the second micro-op of a multi-transfer txn": _transfers_then_finals([[_lt(1), _lt(2)]], [READ]),
    "a repeated id": _transfers_then_finals([[_lt(1), _lt(1), _lt(2)], ALL + [_lt(2)]], [READ]),
    "a phantom id": _transfers_then_finals([ALL + [_lt(9)], ALL], [READ]),
    "an empty final ok lookup": _transfers_then_finals([[], ALL], [READ]),
    "no final reads": _transfers_then_finals([ALL]),
    "no finals at all": _transfers_then_finals([]),
    "unequal final reads and lookups": _transfers_then_finals([ALL, ALL[:2], ALL[::-1], ALL[:2]],
                                                              [READ, READ[:1], READ, [_r(1, 3, None), _r(2)]]),
    "final lookups with nil maps": _transfers_then_finals([[["l-t", 1, None], ["l-t", 2, None], ["l-t", 3, None]],
                                                           [["l-t", 1, None], ["l-t", 2, None], ["l-t", 3, None]],
                                                           [["l-t", 1, None], ["l-t", 2, None], _lt(3, 2, 1)]],
                                                          [[["r", 1, None], ["r", 2, {}]]] * 2),
    "other keywords and tags": _transfers_then_finals([ALL + [["x", 1, None]], ALL + [["y", 1, None]],
                                                       ALL + [["x", 1, None]]], [READ + [["l-t", 5, {}]]]),
    "equal up to formatting": (
        b'{:type :invoke, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 3}]], :process 0, :index 0}\n'
        b'{:type :ok, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 3}]], :process 0, :index 1}\n'
        b'{:type :ok, :process 1, :f :txn, :final? true, :index 2, '
        b':value [[:l-t 1 {:debit-acct 1, :credit-acct 2, :amount 3}]]}\n'
        b'#jepsen.history.Op{:type :ok :process 2 :f :txn :final? true '
        b':value ([:l-t 1N #x {:amount 3 :credit-acct 2N,, :debit-acct 1}])}\n'
        b'{:type :ok, :process 3, :f :txn, :final? :yes, :value [(:l-t   1 {:amount 3, :debit-acct 1, :credit-acct 2})]}\n'
        b'{:type :ok, :process 4, :f :txn, :final? true, :value [[:r 1 {:debits-posted 5, :credits-posted nil}]]}\n'
        b'#jepsen.history.Op{:process 5, :type :ok, :f :txn, :final? 1, '
        b':value [[:r 1 {:credits-posted nil :debits-posted 5N :debits-posted 5}]]}\n'
        b'{:type :ok, :process 6, :f :txn, :final? true, :value [[:r 1 {:debits-posted 5}]]}\n'),
    "one vector": b"[" + _transfers_then_finals([ALL, ALL[:1]], [READ]).replace(b"\n", b"\r\n ") + b"]",
    "empty": b"",
}
# inputs the device refuses (the checkers then parse the file): comments, maps and micro-ops outside the digest's
# reach, and the stock bank's :f spelling
REFUSED_CASES = {
    "comment": b"; a comment\n" + HAND_CASES["valid finals"],
    "unknown key in a final read": _transfers_then_finals([ALL], [[["r", 1, {"debits-posted": 1, "foo": 2}]]]),
    "string key in a final read": _transfers_then_finals([ALL], [[["r", 1, {"debits-posted": 1}]]]).replace(
        b":debits-posted 1}", b':debits-posted 1, "credits-posted" 2}'),
    "4-element micro-op in a final read": _transfers_then_finals([ALL], [[["r", 1, {"debits-posted": 1}, 7]]]),
    "float in a final value": _transfers_then_finals([ALL], [READ]).replace(b":debits-posted 3,", b":debits-posted 3.5,"),
    "f read": b'{:type :invoke, :f :read, :value nil, :process 0}\n{:type :ok, :f :read, :value {1 2}, :process 0}\n',
    "string tag in a final lookup": _transfers_then_finals([ALL + [["x", 1, None]]]).replace(b"[:x 1 nil]",
                                                                                            b'["x" 1 nil]'),
}
