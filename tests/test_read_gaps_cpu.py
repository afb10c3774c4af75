"""The read-gap check without a GPU: hand KATs for every kind against both CPU deciders (the regrouped read pair that
K7, K8, K9, K10 and :SI pass, DOUBLE, a negative Delta, Delta = 0, gap 0, committed and lookup-excluded :info
transfers, a partial read), the caps and the node budget, the input errors, 2,000 random tiny histories (RG_BRUTE ==
RG_SEARCH on every gap RG_SEARCH decides, soundness against the brute-force search for a serial explanation), EDN, the
checker maps and the ABI images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, edn
from jepsen_tigerbeetle_b200 import history as H
from test_monotonic_cpu import inv_r, rd
from test_transfer_lookups_cpu import explainable, final, flat, inv_l, lk, ops_idx, random_tiny, tr


def both(h, max_nodes=0):
    """RG_BRUTE and RG_SEARCH must give every gap RG_SEARCH decides the same code; returns RG_SEARCH's result."""
    b = M.check_read_gaps(h, M.RG_BRUTE, per_gap=True)
    s = M.check_read_gaps(h, M.RG_SEARCH, max_nodes=max_nodes, per_gap=True)
    for x, y in zip(b["per_gap"], s["per_gap"]):
        assert y == 3 or x == y, (b["per_gap"], s["per_gap"])
    return s


def shard(ops):
    return both(flat(ops))["shards"][0]


def witness(s):
    return (s["witness_index"], s["lower_index"], s["kind"], s["key"], s["delta"], s["transfer_id"],
            s["other_index"], s["n_eligible"])


def two(v):
    """A read of accounts 1 and 2 after v moved from 1 to 2."""
    return {1: (v, 0), 2: (0, v)}


# three :info transfers 1 -> 2 of 3, 4 and 5, concurrent with two reads showing 5, then 7: each read alone is explained
# (r1 = {5}, r2 = {3, 4}), but no transfer set grows from 5 to 7
REGROUPED = [tr(0, "invoke", 1, 2, 3, 1), tr(1, "invoke", 1, 2, 4, 2), tr(2, "invoke", 1, 2, 5, 3),
             inv_r(3, [1, 2]), rd(3, two(5)), inv_r(3, [1, 2]), rd(3, two(7)),
             tr(0, "info", 1, 2, 3, 1), tr(1, "info", 1, 2, 4, 2), tr(2, "info", 1, 2, 5, 3)]


def test_regrouped_is_key_and_passes_every_other_check():
    h = flat(REGROUPED)
    r = both(h)
    s = r["shards"][0]
    assert s["valid"] == H.INVALID and s["count_by_kind"] == [1, 0, 0] and s["n_explained"] == 1
    assert witness(s) == (6, 4, abi.RG_KEY, H.counter_key(1, 0), 2, 0, -1, 0)
    b = M.check_read_gaps(h, M.RG_BRUTE)["shards"][0]
    assert (b["valid"], b["kind"], b["key"], b["delta"], b["witness_index"]) == (H.INVALID, abi.RG_KEY,
                                                                                H.counter_key(1, 0), 2, 6)
    assert M.check_monotonic_keys(h)["valid"] == H.VALID
    assert M.check_counter_bounds(h)["valid"] == H.VALID
    assert M.check_transfer_lookups(h)["valid"] == H.VALID
    assert M.check_read_explanations(h)["valid"] == H.VALID
    bank = H.flatten_ops(ops_idx(REGROUPED), "bank")
    from oracle import check_bank_totals
    assert check_bank_totals(bank, H.make_model(H.MODEL_BANK, accounts=range(1, 3)), 0)["valid"] == H.VALID


def test_transfer_forced_into_two_gaps_is_double():
    """One :ok transfer of 5 concurrent with two reads showing 5 and 10: each gap alone is explained by it."""
    ops = [tr(0, "invoke", 1, 2, 5, 9), inv_r(1, [1, 2]), rd(1, two(5)), inv_r(1, [1, 2]), rd(1, two(10)),
           tr(0, "ok", 1, 2, 5, 9)]
    s = shard(ops)
    assert s["valid"] == H.INVALID and s["count_by_kind"] == [0, 0, 1] and s["n_explained"] == 2
    assert witness(s) == (4, 2, abi.RG_DOUBLE, -1, 0, 9, 2, 1)
    assert M.check_read_gaps(flat(ops), M.RG_BRUTE)["shards"][0]["kind"] == abi.RG_DOUBLE


def test_negative_delta_is_key():
    """K7's crossed pair: r1 shows t1 and not t2, r2 the other way round."""
    ops = [tr(0, "invoke", 1, 2, 3, 1), tr(1, "invoke", 3, 4, 4, 2), inv_r(2, [1, 2, 3, 4]),
           rd(2, {1: (3, 0), 2: (0, 3), 3: (0, 0), 4: (0, 0)}), inv_r(3, [1, 2, 3, 4]),
           rd(3, {1: (0, 0), 2: (0, 0), 3: (4, 0), 4: (0, 4)}), tr(0, "ok", 1, 2, 3, 1), tr(1, "ok", 3, 4, 4, 2)]
    s = shard(ops)
    assert witness(s) == (5, 3, abi.RG_KEY, H.counter_key(1, 0), -3, 0, -1, 0)
    assert M.check_monotonic_keys(flat(ops))["valid"] == H.INVALID


def test_zero_delta_is_explained_without_nodes():
    ops = [tr(0, "invoke", 1, 2, 3, 1), tr(0, "ok", 1, 2, 3, 1), inv_r(1, [1, 2]), rd(1, two(3)),
           inv_r(1, [1, 2]), rd(1, two(3))]
    r = both(flat(ops))
    assert (r["valid"], r["n_explained"], r["nodes"]) == (H.VALID, 2, 1)   # gap 0: the root forces t1 in


def test_gap_zero():
    """The first read in the order is explained from the zero state, whatever its invocation."""
    ops = [tr(0, "invoke", 1, 2, 3, 1), tr(0, "ok", 1, 2, 3, 1), inv_r(1, [1, 2]), rd(1, two(2))]
    assert witness(shard(ops)) == (3, -1, abi.RG_KEY, H.counter_key(1, 0), 2, 0, -1, 0)
    ops[3] = rd(1, two(3))
    assert shard(ops)["valid"] == H.VALID


def test_committed_info_transfer_explains_one_gap():
    """A committed :info transfer stays eligible for every later gap, but the amount filter drops it where Delta is
    smaller: only the :info transfer of 2 can close the last gap."""
    ops = [tr(0, "invoke", 1, 2, 4, 1), tr(0, "info", 1, 2, 4, 1), inv_r(1, [1, 2]), rd(1, two(4)),
           tr(2, "invoke", 1, 2, 2, 2), tr(2, "info", 1, 2, 2, 2), inv_r(1, [1, 2]), rd(1, two(6)),
           final(inv_l(3)), final(lk(3, [(1, 1, 2, 4), (2, 1, 2, 2)]))]
    r = both(flat(ops))
    assert (r["valid"], r["n_explained"]) == (H.VALID, 2)


def test_info_transfer_a_later_lookup_lacks_cannot_explain_a_gap():
    ops = [tr(0, "invoke", 1, 2, 4, 1), tr(0, "info", 1, 2, 4, 1), inv_r(1, [1, 2]), rd(1, two(4))]
    assert shard(ops)["valid"] == H.VALID
    s = shard(ops + [final(inv_l(2)), final(lk(2, []))])
    assert witness(s) == (3, -1, abi.RG_KEY, H.counter_key(1, 0), 4, 0, -1, 0)


def test_partial_read_shard_is_unknown():
    ops = [tr(0, "invoke", 1, 2, 2, 1), inv_r(1, [1, 2]), rd(1, two(2)), inv_r(1, [2]),
           {"type": "ok", "process": 1, "f": "txn", "value": [["r", 2, {"debits-posted": 0, "credits-posted": 1}]]},
           tr(0, "ok", 1, 2, 2, 1)]
    r = both(flat(ops))
    s = r["shards"][0]
    assert (s["valid"], s["cause"], s["n_reads"], s["n_explained"], s["nodes"]) == (
        H.UNKNOWN, abi.CAUSE_PARTIAL_READ, 2, 0, 0)
    assert r["per_gap"] == [3, 3]


def _ones(n, shows):
    """n concurrent transfers 1 -> 2 of amount 1 and one read showing shows = (debits of 1, credits of 2)."""
    ops = [tr(p, "invoke", 1, 2, 1, p + 1) for p in range(n)]
    ops += [inv_r(n, [1, 2]), rd(n, {1: (shows[0], 0), 2: (0, shows[1])})]
    return ops + [tr(p, "ok", 1, 2, 1, p + 1) for p in range(n)]


def test_caps():
    r = M.check_read_gaps(flat(_ones(130, (65, 65))))   # more than 128 eligible transfers under Delta
    assert (r["valid"], r["n_undecided"], r["nodes"]) == (H.UNKNOWN, 1, 0)
    # the amount filter runs before the cap: 130 transfers of 2 and three of 1 under Delta = 1 leave three
    amounts = [2] * 130 + [1] * 3
    ops = [tr(p, "invoke", 1, 2, a, p + 1) for p, a in enumerate(amounts)] + [inv_r(133, [1, 2]), rd(133, two(1))]
    r = M.check_read_gaps(flat(ops + [tr(p, "ok", 1, 2, a, p + 1) for p, a in enumerate(amounts)]))
    assert (r["valid"], r["n_explained"]) == (H.VALID, 1)
    assert M.check_read_explanations(flat(ops))["n_undecided"] == 1
    r = M.check_read_gaps(flat(_ones(70, (35, 35))))   # 70 free after the root pruning
    assert (r["valid"], r["n_undecided"], r["nodes"]) == (H.UNKNOWN, 1, 1)
    assert M.check_read_gaps(flat(_ones(40, (20, 20))))["n_explained"] == 1
    # more than 256 keys: every gap is undecided
    accts = list(range(1, 130))
    ops = [inv_r(0, accts), rd(0, {a: (0, 0) for a in accts})]
    assert M.check_read_gaps(flat(ops))["n_undecided"] == 1
    assert M.check_read_gaps(flat(ops), M.RG_BRUTE)["n_explained"] == 1


def test_node_budget_makes_a_gap_undecided():
    # 20 on one side and 21 on the other: pruning cannot see it, the search would need ~C(40, 20) nodes
    h = flat(_ones(40, (20, 21)))
    r = M.check_read_gaps(h)
    assert (r["valid"], r["n_undecided"], r["nodes"]) == (H.UNKNOWN, 1, abi.RG_DEFAULT_MAX_NODES + 1)
    for mx in (1, 2, 100):
        assert M.check_read_gaps(h, max_nodes=mx)["nodes"] == mx + 1
    assert M.check_read_gaps(flat(_ones(40, (41, 41))))["shards"][0]["count_by_kind"] == [1, 0, 0]


def test_errors():
    def raises(ops, match, mutate=None, **kw):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(RuntimeError, match=match):
            M.check_read_gaps(h, **kw)

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", 1, 1 << 30, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, -1))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(0, "ok", 1, 2, 1, 1), inv_l(1), lk(1, [(1, 1, 2, 1)])], "multiple of 5",
           lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "payload", lambda h: h.payload_len.__setitem__(1, 5))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "reserved", flags=1)


# ---- random tiny histories --------------------------------------------------------------------------------------
def test_random_tiny_histories():
    """RG_BRUTE == RG_SEARCH gap for gap; INVALID (by either decider) => no serial explanation.  These histories (at most
    six ops) never give two reads a transfer to share, so none is INVALID here while K7, K8, K9 and K10 all pass it
    (none in 20,000 either); the regrouped KAT above is that case."""
    rng = np.random.default_rng(53)
    verdicts = {H.VALID: 0, H.INVALID: 0, H.UNKNOWN: 0}
    kinds = set()
    for _ in range(2000):
        ops, recs = random_tiny(rng)
        h = flat(ops)
        r = both(h)
        s = r["shards"][0]
        verdicts[s["valid"]] += 1
        kinds.add(s["kind"])
        if s["valid"] == H.INVALID or M.check_read_gaps(h, M.RG_BRUTE)["valid"] == H.INVALID:
            assert not explainable(recs), ops
    assert verdicts[H.VALID] > 200 and verdicts[H.INVALID] > 200, verdicts
    assert kinds >= {0, abi.RG_KEY}, kinds


# ---- EDN ----------------------------------------------------------------------------------------------------------
def test_edn_regrouped_history():
    t = "{:debit-acct 1, :credit-acct 2, :amount %d}"
    r = "[[:r 1 {:debits-posted %d, :credits-posted 0}] [:r 2 {:debits-posted 0, :credits-posted %d}]]"
    lines = [f"{{:type :invoke, :f :txn, :value [[:t {i} {t % a}]], :process {p}, :index {p}}}"
             for p, (i, a) in enumerate([(1, 3), (2, 4), (3, 5)])]
    lines += ["{:type :invoke, :f :txn, :value [[:r 1 nil] [:r 2 nil]], :process 3, :index 3}",
              f"{{:type :ok, :f :txn, :value {r % (5, 5)}, :process 3, :index 4}}",
              "{:type :invoke, :f :txn, :value [[:r 1 nil] [:r 2 nil]], :process 3, :index 5}",
              f"{{:type :ok, :f :txn, :value {r % (7, 7)}, :process 3, :index 6}}"]
    lines += [f"{{:type :info, :f :txn, :value [[:t {i} {t % a}]], :process {p}, :index {7 + p}}}"
              for p, (i, a) in enumerate([(1, 3), (2, 4), (3, 5)])]
    h = H.flatten_ops(edn.read_history("\n".join(lines)), "ledger-lookups")
    g = flat(REGROUPED)
    for name in ("type", "f", "process", "index", "payload_off", "payload_len", "payload"):
        assert np.array_equal(getattr(h, name), getattr(g, name)), name
    assert both(h)["shards"][0]["kind"] == abi.RG_KEY


# ---- checker maps -------------------------------------------------------------------------------------------------
class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_read_gaps(self, h, max_nodes=0):
        return M.check_read_gaps(h, max_nodes=max_nodes)


def test_checker_result_map():
    r = checker.read_gap_checker(ctx=_FakeCtx()).check({}, ops_idx(REGROUPED))
    assert r["valid?"] is False and r["errors"] == {"key": 1} and r["op"] == {"index": 6}
    assert r["lower-op"] == {"index": 4}
    assert (r["read-count"], r["transfer-count"], r["explained-count"], r["undecided-count"], r["error-count"]) == (
        2, 3, 1, 0, 1)
    assert r["error"] == {"type": "key", "eligible-count": 0, "key": [1, "debits-posted"], "delta": 2}
    ops = ops_idx([tr(0, "invoke", 1, 2, 5, 9), inv_r(1, [1, 2]), rd(1, two(5)), inv_r(1, [1, 2]), rd(1, two(10)),
                   tr(0, "ok", 1, 2, 5, 9)])
    r = checker.read_gap_checker(ctx=_FakeCtx()).check({}, ops)
    assert r["error"] == {"type": "double", "eligible-count": 1, "transfer-id": 9, "other-op": {"index": 2}}
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, read_gaps=True)
    assert "read-gaps" in comp.checkers
    assert "read-gaps" not in checker.ledger_checker(linear=False).checkers
    ind = checker.independent_checker(checker.read_gap_checker(ctx=_FakeCtx()))
    assert ind._model() == "ledger-lookups"
    assert checker.read_gap_checker({"max-nodes": 7}, ctx=_FakeCtx()).max_nodes == 7


# ---- ABI ------------------------------------------------------------------------------------------------------
def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(17) == ctypes.sizeof(abi.CRgShard) == 104
    assert lib.jtb_struct_size(18) == ctypes.sizeof(abi.CRgResult) == 80


def test_jni_shim_reports_errors_without_a_device():
    fj = _rg_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_read_gaps(0, fj.jhistory(flat(REGROUPED)), 0), np.int64)


def _rg_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_rg.c (the driver of checkReadGaps)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_rg", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_rg.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_rg.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_rg.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_read_gaps.restype = C.c_void_p
    L.fj_check_read_gaps.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong]
    return fj
