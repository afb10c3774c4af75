"""The read-explanation check without a GPU: hand KATs for both kinds against both CPU deciders, the budget, the input
errors, 2,000 random tiny histories (RX_BRUTE == RX_SEARCH on every read RX_SEARCH decides, soundness against the
brute-force search for a serial explanation, K8 INVALID => K10 INVALID), the synthetic read mutations, EDN, the checker
maps and the ABI images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, edn, synth
from jepsen_tigerbeetle_b200 import history as H
from test_monotonic_cpu import inv_r, rd
from test_transfer_lookups_cpu import explainable, final, flat, inv_l, lk, ops_idx, random_tiny, tr

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_explained", "n_unexplained", "n_undecided", "nodes",
          "shards")


def both(h, max_nodes=0):
    """RX_BRUTE and RX_SEARCH must give every read RX_SEARCH decides the same code; returns RX_SEARCH's result."""
    b = M.check_read_explanations(h, M.RX_BRUTE, per_read=True)
    s = M.check_read_explanations(h, M.RX_SEARCH, max_nodes=max_nodes, per_read=True)
    for x, y in zip(b["per_read"], s["per_read"]):
        assert y == 3 or x == y, (b["per_read"], s["per_read"])
    return s


def shard(ops, model="ledger-lookups"):
    return both(flat(ops, model))["shards"][0]


def witness(s):
    return (s["witness_index"], s["kind"], s["key"], s["n_must"], s["n_may"], s["value"], s["must_sum"])


# transfers 1 -> 2 (t1) and 3 -> 4 (t2), amount 3, both concurrent with a read of accounts 1-4
def torn(shows):
    return [tr(0, "invoke", 1, 2, 3, 1), tr(1, "invoke", 3, 4, 3, 2), inv_r(2, [1, 2, 3, 4]), rd(2, shows),
            tr(0, "ok", 1, 2, 3, 1), tr(1, "ok", 3, 4, 3, 2)]


TORN_PAIR = torn({1: (3, 0), 2: (0, 0), 3: (0, 0), 4: (0, 3)})   # t1's debit half, t2's credit half


def test_torn_pair_is_joint_and_passes_every_other_check():
    h = flat(TORN_PAIR)
    s = both(h)["shards"][0]
    assert s["valid"] == H.INVALID and s["count_by_kind"] == [0, 1]
    assert s["kind"] == abi.RX_JOINT and s["witness_index"] == 3 and (s["n_must"], s["n_may"]) == (0, 0)
    assert s["key"] == H.counter_key(1, 0)   # the root pruning drops both, then debits of 1 cannot reach 3
    assert M.check_counter_bounds(h)["valid"] == H.VALID
    assert M.check_transfer_lookups(h)["valid"] == H.VALID
    assert M.check_monotonic_keys(h)["valid"] == H.VALID
    bank = H.flatten_ops(ops_idx(TORN_PAIR), "bank")
    m = H.make_model(H.MODEL_BANK, accounts=range(1, 5))
    from oracle import check_bank_totals
    assert check_bank_totals(bank, m, 0)["valid"] == H.VALID   # :SI: the totals still sum to zero


def test_single_torn_transfer_is_joint():
    ops = torn({1: (3, 0), 2: (0, 0), 3: (0, 0), 4: (0, 0)})
    s = shard(ops)
    assert s["kind"] == abi.RX_JOINT and s["count_by_kind"] == [0, 1]
    bank = H.flatten_ops(ops_idx(ops), "bank")
    from oracle import check_bank_totals
    r = check_bank_totals(bank, H.make_model(H.MODEL_BANK, accounts=range(1, 5)), 0)
    assert r["valid"] == H.INVALID and r["first_error_type"] == abi.BANK_WRONG_TOTAL


def test_amount_no_subset_produces_is_key():
    """Two concurrent transfers 1 -> 2 of amount 2; the read shows +1 on both sides: inside K8's [0, 4]."""
    ops = [tr(0, "invoke", 1, 2, 2, 1), tr(1, "invoke", 1, 2, 2, 2), inv_r(2, [1, 2]), rd(2, {1: (1, 0), 2: (0, 1)}),
           tr(0, "ok", 1, 2, 2, 1), tr(1, "ok", 1, 2, 2, 2)]
    s = shard(ops)
    assert witness(s) == (3, abi.RX_KEY, H.counter_key(1, 0), 0, 0, 1, 0) and s["count_by_kind"] == [1, 0]
    assert M.check_counter_bounds(flat(ops))["valid"] == H.VALID


def test_survey_b42_is_key():
    """SURVEY B42: a read that misses a transfer completed before it was invoked."""
    ops = [tr(0, "invoke", 1, 2, 5, 1), tr(0, "ok", 1, 2, 5, 1), inv_r(1, [1, 2]), rd(1, {1: (0, 0), 2: (0, 0)})]
    s = shard(ops)
    assert witness(s) == (3, abi.RX_KEY, H.counter_key(1, 0), 1, 0, 0, 5)


def test_committed_info_transfer_explains_a_read():
    ops = [tr(0, "invoke", 1, 2, 4, 1), tr(0, "info", 1, 2, 4, 1), inv_r(1, [1, 2]), rd(1, {1: (4, 0), 2: (0, 4)}),
           final(inv_l(2)), final(lk(2, [(1, 1, 2, 4)]))]
    s = shard(ops)
    assert (s["valid"], s["n_explained"]) == (H.VALID, 1)


def test_info_transfer_a_later_lookup_lacks_cannot_explain_a_read():
    ops = [tr(0, "invoke", 1, 2, 4, 1), tr(0, "info", 1, 2, 4, 1), inv_r(1, [1, 2]), rd(1, {1: (4, 0), 2: (0, 4)})]
    assert shard(ops)["valid"] == H.VALID
    s = shard(ops + [final(inv_l(2)), final(lk(2, []))])
    assert witness(s) == (3, abi.RX_KEY, H.counter_key(1, 0), 0, 0, 4, 0)


def test_partial_read():
    ops = [tr(0, "invoke", 1, 2, 2, 1), inv_r(1, [2]), {"type": "ok", "process": 1, "f": "txn",
                                                        "value": [["r", 2, {"debits-posted": 0, "credits-posted": 2}]]},
           tr(0, "ok", 1, 2, 2, 1)]
    h = flat(ops)
    assert h.payload_len[2] == 6
    assert both(h)["shards"][0]["n_explained"] == 1
    ops[2]["value"][0][2]["credits-posted"] = 1
    assert shard(ops)["kind"] == abi.RX_KEY


def test_more_than_64_free_candidates_is_undecided():
    n = 70
    ops = [tr(p, "invoke", 1, 2, 1, p + 1) for p in range(n)] + [inv_r(n, [1, 2]), rd(n, {1: (n // 2, 0), 2: (0, n // 2)})]
    ops += [tr(p, "ok", 1, 2, 1, p + 1) for p in range(n)]
    h = flat(ops)
    s = M.check_read_explanations(h)
    assert (s["valid"], s["n_undecided"], s["nodes"]) == (H.UNKNOWN, 1, 1)
    assert s["shards"][0]["witness_index"] == -1
    # 40 equal candidates, 20 needed: the search finds one at once
    ops = [tr(p, "invoke", 1, 2, 1, p + 1) for p in range(40)] + [inv_r(40, [1, 2]), rd(40, {1: (20, 0), 2: (0, 20)})]
    ops += [tr(p, "ok", 1, 2, 1, p + 1) for p in range(40)]
    h = flat(ops)
    assert M.check_read_explanations(h)["n_explained"] == 1
    # 20 on one side and 21 on the other: pruning cannot see it, the search would need ~C(40, 20) nodes
    ops[41] = rd(40, {1: (20, 0), 2: (0, 21)})
    r = M.check_read_explanations(flat(ops))
    assert (r["valid"], r["n_undecided"], r["nodes"]) == (H.UNKNOWN, 1, abi.RX_DEFAULT_MAX_NODES + 1)
    ops[41] = rd(40, {1: (41, 0), 2: (0, 41)})
    assert M.check_read_explanations(flat(ops))["shards"][0]["count_by_kind"] == [1, 0]


def test_node_budget_makes_a_read_undecided():
    # amounts 3 and 2 on one key, 7 needed on the other: pruning cannot settle it, the search refutes it
    ops = [tr(p, "invoke", 1, 2, 3 if p < 6 else 2, p + 1) for p in range(12)]
    ops += [inv_r(12, [1, 2]), rd(12, {1: (1, 0), 2: (0, 1)})] + [tr(p, "ok", 1, 2, 3 if p < 6 else 2, p + 1)
                                                                   for p in range(12)]
    h = flat(ops)
    full = M.check_read_explanations(h)
    assert full["valid"] == H.INVALID and full["shards"][0]["kind"] == abi.RX_KEY
    for mx in (1, 2):
        r = M.check_read_explanations(h, max_nodes=mx)
        assert r["n_undecided"] + r["n_unexplained"] == 1


def test_errors():
    def raises(ops, match, mutate=None, **kw):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(RuntimeError, match=match):
            M.check_read_explanations(h, **kw)

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
    """RX_BRUTE == RX_SEARCH read for read; unexplained => no serial explanation; K8 INVALID => K10 INVALID on
    histories whose lookups show no :fail or future transfer (K10's must set trusts them, K8 ignores them)."""
    rng = np.random.default_rng(41)
    verdicts = {H.VALID: 0, H.INVALID: 0, H.UNKNOWN: 0}
    kinds = set()
    for _ in range(2000):
        ops, recs = random_tiny(rng)
        h = flat(ops)
        r = both(h)
        s = r["shards"][0]
        verdicts[s["valid"]] += 1
        kinds.add(s["kind"])
        if s["valid"] == H.INVALID:
            assert not explainable(recs), ops
        tl = M.check_transfer_lookups(h)["shards"][0]["count_by_kind"]
        if (M.check_counter_bounds(h)["valid"] == H.INVALID and s["n_undecided"] == 0
                and tl[abi.TL_FAILED_VISIBLE - 1] == tl[abi.TL_FUTURE - 1] == 0):
            assert s["valid"] == H.INVALID, ops
    assert verdicts[H.VALID] > 200 and verdicts[H.INVALID] > 200, verdicts
    assert kinds >= {0, abi.RX_KEY}, kinds


def test_k10_finds_what_k8_cannot():
    """On random tiny histories K10 refutes reads inside K8's bounds."""
    rng = np.random.default_rng(43)
    more = 0
    for _ in range(600):
        h = flat(random_tiny(rng)[0])
        if M.check_counter_bounds(h)["valid"] == H.VALID and M.check_read_explanations(h)["valid"] == H.INVALID:
            more += 1
    assert more > 0


# ---- synthetic histories ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("mutation", ["torn_transfer", "torn_pair", "split_amount"])
def test_read_mutations(mutation):
    spec = synth.SynthSpec("bank", 3000, 16, 3, final_reads=True)
    base = synth.generate_ledger_lookups(spec)
    h = synth.generate_ledger_lookups(spec, **{mutation: True})
    for name in ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_off", "payload_len"):
        assert np.array_equal(getattr(h, name), getattr(base, name)), name
    assert np.count_nonzero(h.payload != base.payload) == (1 if mutation == "torn_transfer" else 2)
    r = M.check_read_explanations(h)
    s = r["shards"][0]
    assert r["valid"] == H.INVALID and s["witness_index"] == h.meta["torn_read_index"], s
    assert M.check_read_explanations(base)["n_unexplained"] == 0
    assert M.check_counter_bounds(h)["valid"] == H.VALID and M.check_transfer_lookups(h)["valid"] == H.VALID


def test_torn_pair_keeps_the_totals():
    spec = synth.SynthSpec("bank", 3000, 16, 3, final_reads=True)
    h = synth.generate_ledger_lookups(spec, torn_pair=True)
    e = int(np.nonzero(h.index == h.meta["torn_read_index"])[0][0])
    v = h.payload[h.payload_off[e]:h.payload_off[e] + h.payload_len[e]].reshape(-1, 3)
    assert int(v[1::2, 1].sum() - v[0::2, 1].sum()) == 0   # credits - debits: the balances still sum to zero
    assert M.check_read_explanations(h)["shards"][0]["kind"] == abi.RX_JOINT


def test_oracle_on_c3_size():
    for kw in ({}, {"lost_transfer": True}):
        h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True), **kw)
        r = M.check_read_explanations(h)
        assert r["n_explained"] + r["n_unexplained"] > 0.75 * r["n_reads"]
        assert (r["n_unexplained"] > 0) == bool(kw)


def test_edn_torn_history():
    text = """
{:type :invoke, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 3}]], :process 0, :index 0}
{:type :invoke, :f :txn, :value [[:t 2 {:debit-acct 3, :credit-acct 4, :amount 3}]], :process 1, :index 1}
{:type :invoke, :f :txn, :value [[:r 1 nil] [:r 2 nil] [:r 3 nil] [:r 4 nil]], :process 2, :index 2}
{:type :ok, :f :txn, :value [[:r 1 {:debits-posted 3, :credits-posted 0}] [:r 2 {:debits-posted 0, :credits-posted 0}] [:r 3 {:debits-posted 0, :credits-posted 0}] [:r 4 {:debits-posted 0, :credits-posted 3}]], :process 2, :index 3}
{:type :ok, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 3}]], :process 0, :index 4}
{:type :ok, :f :txn, :value [[:t 2 {:debit-acct 3, :credit-acct 4, :amount 3}]], :process 1, :index 5}
"""
    h = H.flatten_ops(edn.read_history(text), "ledger-lookups")
    g = flat(TORN_PAIR)
    for name in ("type", "f", "process", "index", "payload_off", "payload_len", "payload"):
        assert np.array_equal(getattr(h, name), getattr(g, name)), name
    assert both(h)["shards"][0]["kind"] == abi.RX_JOINT


# ---- checker maps -------------------------------------------------------------------------------------------------
class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_read_explanations(self, h, max_nodes=0):
        return M.check_read_explanations(h, max_nodes=max_nodes)


def test_checker_result_map():
    r = checker.read_explanation_checker(ctx=_FakeCtx()).check({}, ops_idx(TORN_PAIR))
    assert r["valid?"] is False and r["errors"] == {"joint": 1} and r["op"] == {"index": 3}
    assert (r["read-count"], r["transfer-count"], r["explained-count"], r["undecided-count"], r["error-count"]) == (
        1, 2, 0, 0, 1)
    assert r["error"] == {"type": "joint", "must-count": 0, "may-count": 0, "key": [1, "debits-posted"]}
    ops = ops_idx([tr(0, "invoke", 1, 2, 5, 1), tr(0, "ok", 1, 2, 5, 1), inv_r(1, [1, 2]),
                   rd(1, {1: (0, 0), 2: (0, 0)})])
    r = checker.read_explanation_checker(ctx=_FakeCtx()).check({}, ops)
    assert r["error"] == {"type": "key", "must-count": 1, "may-count": 0, "key": [1, "debits-posted"], "value": 0,
                          "must-sum": 5}
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, read_explanations=True)
    assert "read-explanations" in comp.checkers
    assert "read-explanations" not in checker.ledger_checker(linear=False).checkers
    ind = checker.independent_checker(checker.read_explanation_checker(ctx=_FakeCtx()))
    assert ind._model() == "ledger-lookups"
    assert checker.read_explanation_checker({"max-nodes": 7}, ctx=_FakeCtx()).max_nodes == 7


# ---- ABI ------------------------------------------------------------------------------------------------------
def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(15) == ctypes.sizeof(abi.CRxShard) == 88
    assert lib.jtb_struct_size(16) == ctypes.sizeof(abi.CRxResult) == 72


def test_jni_shim_reports_errors_without_a_device():
    fj = _rx_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_read_explanations(0, fj.jhistory(flat(TORN_PAIR)), 0), np.int64)


def _rx_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_rx.c (the driver of checkReadExplanations)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_rx", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_rx.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_rx.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_rx.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_read_explanations.restype = C.c_void_p
    L.fj_check_read_explanations.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong]
    return fj
