"""The transfer-placement check without a GPU: the "chained" and "lost behind a crash" KATs that :SI, K7, K8, K9, K10
and K11 all pass, PLACE, DOUBLE in a later round, an incomplete gap holding LOST back, max_rounds, the caps, the node
budget, the input errors, a partial read, random tiny and regrouping histories (TP_SEARCH INVALID => TP_BRUTE INVALID
=> no serial explanation, K11 INVALID => K12 INVALID), EDN, the checker maps and the ABI images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, edn
from jepsen_tigerbeetle_b200 import history as H
from test_monotonic_cpu import inv_r, rd
from test_read_gaps_cpu import _ones, two
from test_transfer_lookups_cpu import explainable, final, flat, inv_l, lk, ops_idx, random_tiny, tr

READER = 99


def script(steps):
    """Ops and brute-force records from steps: ("t", name, amount) invokes a transfer 1 -> 2 on a process of its own,
    ("ok" | "info" | "fail", name) completes it, ("r", v) is a read of accounts 1 and 2 after v moved (invoke and
    completion back to back), ("l", [names]) a lookup returning those transfers."""
    ops, recs, ts = [], [], {}
    for st in steps:
        if st[0] == "t":
            r = {"kind": "t", "inv": len(ops), "comp": None, "fate": None, "a": st[2], "b": 1, "c": 2,
                 "id": len(ts) + 1}
            ts[st[1]] = r
            recs.append(r)
            ops.append(tr(r["id"], "invoke", 1, 2, st[2], r["id"]))
        elif st[0] in ("ok", "info", "fail"):
            r = ts[st[1]]
            r["comp"], r["fate"] = len(ops), st[0]
            ops.append(tr(r["id"], st[0], 1, 2, r["a"], r["id"]))
        elif st[0] == "r":
            v = st[1]
            r = {"kind": "r", "inv": len(ops), "comp": len(ops) + 1, "fate": "ok",
                 "values": {H.counter_key(1, 0): v, H.counter_key(1, 1): 0, H.counter_key(2, 0): 0,
                            H.counter_key(2, 1): v}}
            recs.append(r)
            ops += [inv_r(READER, [1, 2]), rd(READER, two(v))]
        else:
            got = [ts[n] for n in st[1]]
            r = {"kind": "l", "inv": len(ops), "comp": len(ops) + 1, "fate": "ok",
                 "recs": [(t["id"], 1, 2, t["a"]) for t in got]}
            recs.append(r)
            ops += [inv_l(READER), lk(READER, r["recs"])]
    return ops, recs


def tp(h, **kw):
    return M.check_transfer_placement(h, M.TP_SEARCH, **kw)


def witness(s):
    return (s["witness_index"], s["lower_index"], s["kind"], s["key"], s["round"], s["delta"], s["transfer_id"],
            s["other_index"])


def every_other_check_passes(ops):
    h = flat(ops)
    assert M.check_monotonic_keys(h)["valid"] == H.VALID
    assert M.check_counter_bounds(flat(ops, "ledger-counters"))["valid"] == H.VALID
    assert M.check_transfer_lookups(h)["valid"] == H.VALID
    for algo in (M.RX_SEARCH, M.RX_BRUTE):
        assert M.check_read_explanations(h, algo)["valid"] == H.VALID
    for algo in (M.RG_SEARCH, M.RG_BRUTE):
        assert M.check_read_gaps(h, algo)["valid"] == H.VALID
    from oracle import check_bank_totals
    bank = H.flatten_ops(ops_idx(ops), "bank")
    assert check_bank_totals(bank, H.make_model(H.MODEL_BANK, accounts=range(1, 3)), 0)["valid"] == H.VALID


# :info transfers c = 5, a = 3, d = 2, e = 4 and reads of 5, 10, 12: gap 0 can only be {c}, gap 2 only {d}, which leaves
# gap 1 (Delta 5) with {a} = 3
CHAINED = [("t", "c", 5), ("r", 5), ("t", "a", 3), ("t", "d", 2), ("r", 10), ("t", "e", 4), ("r", 12),
           ("info", "c"), ("info", "a"), ("info", "d"), ("info", "e")]
# an :info u = 5 before r1 = 5, then an :ok t = 5, then r2 = 5: t must be in r2's state, but no gap can hold it
LOST = [("t", "u", 5), ("r", 5), ("t", "t", 5), ("ok", "t"), ("r", 5), ("info", "u")]


def test_chained_is_key_in_round_one():
    ops, recs = script(CHAINED)
    h = flat(ops)
    s = tp(h)["shards"][0]
    assert s["valid"] == H.INVALID and s["count_by_kind"] == [1, 0, 0, 0] and s["n_placed"] == 2
    # the witness: the gap closed by r2 (completion :index 6) over r1 (:index 2), key debits of 1, Delta' = 5 - 0
    assert witness(s) == (6, 2, abi.TP_KEY, H.counter_key(1, 0), 1, 5, 0, -1)
    assert tp(h, max_rounds=1)["valid"] == H.VALID
    assert M.check_transfer_placement(h, M.TP_BRUTE)["valid"] == H.INVALID
    every_other_check_passes(ops)
    assert not explainable(recs)


def test_lost_behind_a_crash():
    ops, recs = script(LOST)
    h = flat(ops)
    s = tp(h)["shards"][0]
    assert s["valid"] == H.INVALID and s["count_by_kind"] == [0, 0, 0, 1] and s["n_explained"] == 2
    # LOST at round 0: the read that must hold t (:index 6), the :ok that fixes M(t) (:index 4)
    assert witness(s) == (6, 2, abi.TP_LOST, -1, 0, 0, 2, 4)
    assert M.check_transfer_placement(h, M.TP_BRUTE)["valid"] == H.INVALID
    every_other_check_passes(ops)
    assert not explainable(recs)


def test_place_then_decides_a_gap():
    """An :ok x = 3 must be in r2's state and only gap 1 can hold it; once placed, gap 1 (Delta 5) is Delta' = 2,
    which only the :info y = 2 closes, so y leaves gap 2, where {z} = 4 then explains."""
    ops, _ = script([("t", "x", 3), ("t", "y", 2), ("t", "z", 4), ("r", 0), ("ok", "x"), ("r", 5), ("r", 9),
                     ("info", "y"), ("info", "z")])
    h = flat(ops)
    r = tp(h)
    s = r["shards"][0]
    assert r["valid"] == H.VALID and s["n_placed"] >= 1 and s["rounds"] >= 2
    assert M.check_transfer_placement(h, M.TP_BRUTE)["valid"] == H.VALID


def test_double_in_a_later_round():
    """K11 passes this regrouping history; K12 places three transfers in rounds 0 and 1, after which two gaps both need
    the same one (DOUBLE) and one gap cannot close (KEY, in round 1)."""
    ops, recs = script([("t", "a", 2), ("t", "b", 3), ("t", "c", 2), ("info", "c"), ("r", 4), ("t", "d", 1),
                        ("t", "e", 2), ("ok", "a"), ("ok", "d"), ("r", 6), ("ok", "e"), ("r", 10), ("info", "b")])
    h = flat(ops)
    s = tp(h)["shards"][0]
    assert s["valid"] == H.INVALID and s["count_by_kind"] == [1, 0, 1, 0] and s["n_placed"] == 3
    assert (s["kind"], s["round"]) == (abi.TP_KEY, 1)
    assert M.check_read_gaps(h)["valid"] != H.INVALID
    assert tp(h, max_rounds=1)["n_double"] == 0
    assert M.check_transfer_placement(h, M.TP_BRUTE)["valid"] == H.INVALID
    assert not explainable(recs)


def test_incomplete_gap_holds_lost_back():
    """The lost-behind-a-crash shape, with more than JTB_TP_MAX_GATHER transfers of 1 under gap 1's Delta: that gap
    does not know all its candidates, so t is not LOST."""
    n = abi.TP_MAX_GATHER + 2
    steps = [("t", "u", 5), ("r", 5), ("t", "t", 5), ("ok", "t")] + [("t", f"x{i}", 1) for i in range(n)]
    steps += [("r", 5 + n)] + [("info", f"x{i}") for i in range(n)] + [("info", "u")]
    s = tp(flat(script(steps)[0]))["shards"][0]
    assert s["count_by_kind"][3] == 0 and s["valid"] == H.UNKNOWN


def test_max_rounds_and_defaults():
    h = flat(script(CHAINED)[0])
    assert tp(h)["rounds"] == tp(h, max_rounds=abi.TP_DEFAULT_MAX_ROUNDS)["rounds"] == 2   # round 1 places nothing
    assert tp(h, max_rounds=2)["rounds"] == 2 and tp(h, max_rounds=2)["valid"] == H.INVALID
    one = tp(h, max_rounds=1)
    assert one["rounds"] == 1 and one["n_placed"] == 2


def test_max_rounds_one_has_k11s_gap_fields():
    rng = np.random.default_rng(71)
    for _ in range(300):
        h = flat(random_tiny(rng)[0])
        g, k = tp(h, max_rounds=1), M.check_read_gaps(h)
        for a, b in zip(g["shards"], k["shards"]):
            assert (a["n_explained"], a["n_undecided"], a["count_by_kind"][:3], a["nodes"]) == (
                b["n_explained"], b["n_undecided"], b["count_by_kind"], b["nodes"])


def test_caps_and_node_budget():
    r = tp(flat(_ones(130, (65, 65))))
    assert (r["valid"], r["n_undecided"], r["nodes"]) == (H.UNKNOWN, 1, 0)
    r = tp(flat(_ones(70, (35, 35))))
    assert (r["valid"], r["n_undecided"]) == (H.UNKNOWN, 1)
    h = flat(_ones(40, (20, 21)))
    assert tp(h)["n_undecided"] == 1
    for mx in (1, 2, 100):
        assert tp(h, max_nodes=mx)["nodes"] == tp(h, max_nodes=mx, max_rounds=1)["nodes"] * 2
    accts = list(range(1, 130))
    assert tp(flat([inv_r(0, accts), rd(0, {a: (0, 0) for a in accts})]))["n_undecided"] == 1


def test_partial_read_shard_is_unknown():
    ops = [tr(0, "invoke", 1, 2, 2, 1), inv_r(1, [1, 2]), rd(1, two(2)), inv_r(1, [2]),
           {"type": "ok", "process": 1, "f": "txn", "value": [["r", 2, {"debits-posted": 0, "credits-posted": 1}]]},
           tr(0, "ok", 1, 2, 2, 1)]
    s = tp(flat(ops))["shards"][0]
    assert (s["valid"], s["cause"], s["n_reads"], s["rounds"], s["nodes"]) == (H.UNKNOWN, abi.CAUSE_PARTIAL_READ, 2,
                                                                              0, 0)


def test_errors():
    def raises(ops, match, mutate=None, **kw):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(RuntimeError, match=match):
            M.check_transfer_placement(h, **kw)

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", 1, 1 << 30, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, -1))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(0, "ok", 1, 2, 1, 1), inv_l(1), lk(1, [(1, 1, 2, 1)])], "multiple of 5",
           lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "payload", lambda h: h.payload_len.__setitem__(1, 5))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "reserved", flags=1)


# ---- random histories ---------------------------------------------------------------------------------------------
def regrouping(rng):
    """One account pair, 2-4 sequential reads and 1-5 concurrent :ok / :info transfers; each read shows a subset-sum of
    the transfers invoked before it, drawn independently of the other reads, so the read states often do not nest."""
    steps, invoked, open_ = [], [], []
    n_t, n_r = int(rng.integers(1, 6)), int(rng.integers(2, 5))
    events = ["t"] * n_t + ["r"] * n_r
    rng.shuffle(events)
    for e in events:
        if e == "t":
            name = f"t{len(invoked)}"
            steps.append(("t", name, int(rng.integers(1, 4))))
            invoked.append(steps[-1])
            open_.append(name)
        else:
            for name in list(open_):
                if rng.random() < 0.4:
                    steps.append((str(rng.choice(["ok", "info"])), name))
                    open_.remove(name)
            steps.append(("r", int(sum(t[2] for t in invoked if rng.random() < 0.5))))
    steps += [(str(rng.choice(["ok", "info"])), name) for name in open_]
    return script(steps)


@pytest.mark.parametrize("gen", ["tiny", "regrouping"])
def test_random_histories(gen):
    rng = np.random.default_rng(83 if gen == "tiny" else 89)
    counts = {"search": 0, "brute": 0, "k11": 0}
    for _ in range(2000):
        ops, recs = random_tiny(rng) if gen == "tiny" else regrouping(rng)
        h = flat(ops)
        s = tp(h)["valid"]
        b = M.check_transfer_placement(h, M.TP_BRUTE)["valid"]
        k = M.check_read_gaps(h)["valid"]
        if s == H.INVALID:
            assert b == H.INVALID, ops
        if b == H.INVALID:
            assert not explainable(recs), ops
        if k == H.INVALID:
            assert s == H.INVALID, ops
        counts["search"] += s == H.INVALID and b == H.INVALID
        counts["brute"] += b == H.INVALID
        counts["k11"] += k == H.INVALID and b == H.INVALID
    print(f"{gen}: TP_SEARCH catches {counts['search']} of {counts['brute']} TP_BRUTE-INVALID histories "
          f"(K11: {counts['k11']})")
    assert counts["brute"] > 0


# ---- EDN ----------------------------------------------------------------------------------------------------------
def test_edn_lost_history():
    ops, _ = script(LOST)
    t = "[[:t {i} {{:debit-acct 1, :credit-acct 2, :amount 5}}]]"
    r = "[[:r 1 {:debits-posted 5, :credits-posted 0}] [:r 2 {:debits-posted 0, :credits-posted 5}]]"
    rinv = "[[:r 1 nil] [:r 2 nil]]"
    lines = [f"{{:type :invoke, :f :txn, :value {t.format(i=1)}, :process 1, :index 0}}",
             f"{{:type :invoke, :f :txn, :value {rinv}, :process 99, :index 1}}",
             f"{{:type :ok, :f :txn, :value {r}, :process 99, :index 2}}",
             f"{{:type :invoke, :f :txn, :value {t.format(i=2)}, :process 2, :index 3}}",
             f"{{:type :ok, :f :txn, :value {t.format(i=2)}, :process 2, :index 4}}",
             f"{{:type :invoke, :f :txn, :value {rinv}, :process 99, :index 5}}",
             f"{{:type :ok, :f :txn, :value {r}, :process 99, :index 6}}",
             f"{{:type :info, :f :txn, :value {t.format(i=1)}, :process 1, :index 7}}"]
    h = H.flatten_ops(edn.read_history("\n".join(lines)), "ledger-lookups")
    g = flat(ops)
    for name in ("type", "f", "process", "index", "payload_off", "payload_len", "payload"):
        assert np.array_equal(getattr(h, name), getattr(g, name)), name
    assert tp(h)["shards"][0]["kind"] == abi.TP_LOST


# ---- checker maps -------------------------------------------------------------------------------------------------
class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_transfer_placement(self, h, max_nodes=0, max_rounds=0):
        return M.check_transfer_placement(h, max_nodes=max_nodes, max_rounds=max_rounds)


def test_checker_result_map():
    r = checker.transfer_placement_checker(ctx=_FakeCtx()).check({}, ops_idx(script(LOST)[0]))
    assert r["valid?"] is False and r["errors"] == {"lost": 1} and r["op"] == {"index": 6}
    assert r["lower-op"] == {"index": 2}
    assert (r["read-count"], r["transfer-count"], r["explained-count"], r["undecided-count"], r["error-count"],
            r["placed-count"], r["rounds"]) == (2, 2, 2, 0, 1, 1, 2)
    assert r["error"] == {"type": "lost", "round": 0, "eligible-count": 0, "transfer-id": 2,
                          "other-op": {"index": 4}}
    r = checker.transfer_placement_checker(ctx=_FakeCtx()).check({}, ops_idx(script(CHAINED)[0]))
    assert r["error"] == {"type": "key", "round": 1, "eligible-count": 1, "key": [1, "debits-posted"], "delta": 5}
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, transfer_placement=True)
    assert "transfer-placement" in comp.checkers
    assert "transfer-placement" not in checker.ledger_checker(linear=False).checkers
    ind = checker.independent_checker(checker.transfer_placement_checker(ctx=_FakeCtx()))
    assert ind._model() == "ledger-lookups"
    c = checker.transfer_placement_checker({"max-nodes": 7, "max-rounds": 3}, ctx=_FakeCtx())
    assert (c.max_nodes, c.max_rounds) == (7, 3)


# ---- ABI ------------------------------------------------------------------------------------------------------
def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(19) == ctypes.sizeof(abi.CTpShard) == 128
    assert lib.jtb_struct_size(20) == ctypes.sizeof(abi.CTpResult) == 104


def test_jni_shim_reports_errors_without_a_device():
    fj = _tp_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_transfer_placement(0, fj.jhistory(flat(script(LOST)[0])), 0, 0), np.int64)


def _tp_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_tp.c (the driver of checkTransferPlacement)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_tp", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_tp.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_tp.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_tp.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_transfer_placement.restype = C.c_void_p
    L.fj_check_transfer_placement.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong, C.c_int]
    return fj
