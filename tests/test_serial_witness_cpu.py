"""The serial-witness check without a GPU: SW_SEARCH on 2,000 random tiny and 2,000 regrouping histories (every VALID
passes the independent verifier, has a serial explanation and is VALID for the bank model's :linear), one hand case
per cause, the checker maps and the ABI images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker
from jepsen_tigerbeetle_b200 import history as H
from serial_witness import verify
from test_monotonic_cpu import inv_r, rd
from test_read_gaps_cpu import _ones, two
from test_transfer_lookups_cpu import explainable, flat, ops_idx, random_tiny, tr
from test_transfer_placement_cpu import CHAINED, LOST, regrouping, script


def sw(h, **kw):
    r = M.check_serial_witness(h, **kw)
    verify(h, r)
    return r


# :info x = 2, y = 1, z = 1 and reads of 2, 4: both gaps choose {x} in round 0; the smaller one keeps it, and the
# larger one takes {y, z} in round 1
CONFLICT = [("t", "x", 2), ("t", "y", 1), ("t", "z", 1), ("r", 2), ("r", 4), ("info", "x"), ("info", "y"),
            ("info", "z")]
# the same transfers and reads of 2, 4, 6: every gap explains alone, but after {x} and {y, z} are fixed nothing is
# left for the third gap
CONFLICT_LOST = CONFLICT[:5] + [("r", 6)] + CONFLICT[5:]
# :info x = y = z = 1 and a read of 2: the search branches, so one node leaves the gap undecided
BRANCHING = [("t", "x", 1), ("t", "y", 1), ("t", "z", 1), ("r", 2), ("info", "x"), ("info", "y"), ("info", "z")]
# a long read r1 [0, 4] shows the :info u = 2 (invoked at 3), not the :ok t = 1 (done at 2), and r2 shows both: t
# completed before u was invoked, so no point of r1 can hold u without t
LATE = [inv_r(9, [1, 2]), tr(1, "invoke", 1, 2, 1, 1), tr(1, "ok", 1, 2, 1, 1), tr(2, "invoke", 1, 2, 2, 2),
        rd(9, two(2)), inv_r(9, [1, 2]), rd(9, two(3)), tr(2, "info", 1, 2, 2, 2)]
PARTIAL = [tr(0, "invoke", 1, 2, 2, 1), inv_r(1, [1, 2]), rd(1, two(2)), inv_r(1, [2]), rd(1, {2: (0, 1)}),
           tr(0, "ok", 1, 2, 2, 1)]
# an :ok transfer of amount 0 and one on accounts no read observes: both commit freely; a crashed one never
FREE = [tr(0, "invoke", 1, 2, 0, 1), tr(0, "ok", 1, 2, 0, 1), tr(1, "invoke", 3, 4, 5, 2), tr(1, "ok", 3, 4, 5, 2),
        tr(2, "invoke", 1, 2, 1, 3), inv_r(9, [1, 2]), rd(9, two(0)), tr(2, "info", 1, 2, 1, 3)]
NO_READS = [tr(0, "invoke", 1, 2, 3, 1), tr(0, "ok", 1, 2, 3, 1), tr(1, "invoke", 1, 2, 1, 2), tr(2, "invoke", 2, 1, 1, 3),
            tr(2, "fail", 2, 1, 1, 3)]


def hand_histories():
    """(name, history, keyword arguments, cause) of one history per cause."""
    return [("chained", flat(script(CHAINED)[0]), {}, abi.CAUSE_ANOMALY),
            ("lost behind a crash", flat(script(LOST)[0]), {}, abi.CAUSE_ANOMALY),
            ("branching", flat(script(BRANCHING)[0]), {}, 0),
            ("branching, one node", flat(script(BRANCHING)[0]), {"max_nodes": 1}, abi.CAUSE_UNDECIDED),
            ("partial read", flat(PARTIAL), {}, abi.CAUSE_PARTIAL_READ),
            ("conflict", flat(script(CONFLICT)[0]), {}, 0),
            ("conflict, nothing left", flat(script(CONFLICT_LOST)[0]), {}, abi.CAUSE_NO_WITNESS),
            ("conflict, one round", flat(script(CONFLICT)[0]), {"max_rounds": 1}, abi.CAUSE_NO_WITNESS),
            ("late", flat(LATE), {}, abi.CAUSE_REAL_TIME),
            ("free", flat(FREE), {}, 0),
            ("no reads", flat(NO_READS), {}, 0)]


def test_one_cause_each():
    for name, h, kw, cause in hand_histories():
        s = sw(h, **kw)["shards"][0]
        assert s["cause"] == cause and (s["valid"] == H.VALID) == (cause == 0), (name, s)


def test_conflict_is_resolved_by_the_smaller_gap():
    r = sw(flat(script(CONFLICT)[0]))
    s = r["shards"][0]
    assert (s["valid"], s["rounds"], s["n_committed"], s["n_committed_crashed"], s["n_after"]) == (H.VALID, 2, 3, 3, 0)
    # x in r1's state (completion :index 4), y and z in r2's (:index 6)
    assert r["commit_read"].tolist() == [4, 6, 6]
    s = sw(flat(script(CONFLICT_LOST)[0]))["shards"][0]
    # the third gap (closed by r3, :index 8) has nothing left in round 2
    assert (s["valid"], s["cause"], s["rounds"], s["fail_index"], s["transfer_id"]) == (
        H.UNKNOWN, abi.CAUSE_NO_WITNESS, 3, 8, -1)
    assert M.check_transfer_placement(flat(script(CONFLICT_LOST)[0]))["valid"] == H.VALID


def test_max_rounds():
    h = flat(script(CONFLICT)[0])
    s = sw(h, max_rounds=1)["shards"][0]
    assert (s["cause"], s["rounds"], s["fail_index"]) == (abi.CAUSE_NO_WITNESS, 1, 6)
    assert sw(h, max_rounds=2)["valid"] == H.VALID
    assert sw(h)["rounds"] == sw(h, max_rounds=abi.TP_DEFAULT_MAX_ROUNDS)["rounds"] == 2


def test_real_time_names_the_transfer():
    r = sw(flat(LATE))
    s = r["shards"][0]
    # t (id 1) must follow r1, whose point is at least u's invocation (3), but t completed at :index 2
    assert (s["valid"], s["cause"], s["fail_index"], s["transfer_id"]) == (H.UNKNOWN, abi.CAUSE_REAL_TIME, 2, 1)
    assert r["commit_read"].tolist() == [abi.SW_NEVER, abi.SW_NEVER]
    assert M.check_transfer_placement(flat(LATE))["valid"] == H.VALID


def test_free_never_and_no_reads():
    r = sw(flat(FREE))
    assert r["valid"] == H.VALID and r["commit_read"].tolist() == [abi.SW_FREE, abi.SW_FREE, abi.SW_NEVER]
    r = sw(flat(NO_READS))
    assert (r["valid"], r["n_reads"], r["rounds"]) == (H.VALID, 0, 0)
    assert r["commit_read"].tolist() == [abi.SW_FREE, abi.SW_NEVER, abi.SW_NEVER]


def test_partial_read_and_anomalies_commit_nothing():
    for ops in (PARTIAL, script(CHAINED)[0], script(LOST)[0]):
        r = sw(flat(ops))
        assert r["valid"] == H.UNKNOWN and set(r["commit_read"].tolist()) == {abi.SW_NEVER}
        assert (r["nodes"], r["rounds"], r["n_committed"]) == (0, 0, 0)


def test_undecided_and_caps():
    assert sw(flat(_ones(40, (20, 21))))["shards"][0]["cause"] == abi.CAUSE_UNDECIDED
    assert sw(flat(_ones(130, (65, 65))))["shards"][0]["cause"] == abi.CAUSE_UNDECIDED


def test_errors():
    with pytest.raises(RuntimeError, match="negative amount"):
        M.check_serial_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]))
    with pytest.raises(RuntimeError, match="reserved"):
        M.check_serial_witness(flat([tr(0, "invoke", 1, 2, 1, 1)]), flags=1)


# ---- random histories ---------------------------------------------------------------------------------------------
def lookup_free(recs):
    """The records without lookups, with the crashed transfers' completions dropped: a crashed transfer may commit at
    any point after its invocation (as in knossos and in the witness, which give it cp = infinity)."""
    return [dict(r, comp=None) if r["fate"] == "info" else r for r in recs if r["kind"] != "l"]


def bank_ops(ops):
    """The lookup-free ops (a lookup's invoke and completion both go, as do txns with no micro-ops)."""
    return [o for o in ops if o["value"] and not any(m[0] == "l-t" for m in o["value"])]


# (VALID verdicts of SW_SEARCH, explainable histories) among the 2,000 of each generator (fixed seeds)
PINNED = {"tiny": (1523, 1530), "regrouping": (1066, 1068)}


@pytest.mark.parametrize("gen", ["tiny", "regrouping"])
def test_random_histories(gen, oracle_mod):
    rng = np.random.default_rng(103 if gen == "tiny" else 107)
    model = H.make_model(H.MODEL_BANK, accounts=range(1, 3))
    n_valid = n_explainable = 0
    for _ in range(2000):
        ops, recs = random_tiny(rng) if gen == "tiny" else regrouping(rng)
        h = flat(ops)
        r = sw(h)
        ok = explainable(lookup_free(recs))
        n_explainable += ok
        if r["valid"] != H.VALID:
            continue
        n_valid += 1
        assert ok, ops
        bank = H.flatten_ops(ops_idx(bank_ops(ops)), "bank")
        assert oracle_mod.check_linearizable(bank, model, oracle_mod.ALGO_WGL_COMPACT)["valid"] == H.VALID, ops
    print(f"{gen}: SW_SEARCH proves {n_valid} of the {n_explainable} explainable histories")
    assert (n_valid, n_explainable) == PINNED[gen]


# ---- checker maps -------------------------------------------------------------------------------------------------
class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_serial_witness(self, h, max_nodes=0, max_rounds=0, witness=False):
        return M.check_serial_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, witness=witness)


def test_checker_result_map():
    c = checker.serial_witness_checker(ctx=_FakeCtx())
    r = c.check({}, ops_idx(script(CONFLICT)[0]))
    assert r["valid?"] is True and (r["read-count"], r["transfer-count"], r["committed-count"],
                                    r["committed-crashed-count"], r["after-count"], r["rounds"]) == (2, 3, 3, 3, 0, 2)
    r = c.check({}, ops_idx(LATE))
    assert r["valid?"] == "unknown" and r["cause"] == "real-time"
    assert r["op"] == {"index": 2} and r["transfer-id"] == 1
    r = c.check({}, ops_idx(script(CHAINED)[0]))
    assert r["valid?"] == "unknown" and r["cause"] == "anomaly"
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, serial_witness=True)
    assert "serial-witness" in comp.checkers
    assert "serial-witness" not in checker.ledger_checker(linear=False).checkers
    assert checker.independent_checker(checker.serial_witness_checker(ctx=_FakeCtx()))._model() == "ledger-lookups"
    c = checker.serial_witness_checker({"max-nodes": 7, "max-rounds": 3}, ctx=_FakeCtx())
    assert (c.max_nodes, c.max_rounds) == (7, 3)


# ---- ABI ------------------------------------------------------------------------------------------------------
def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(21) == ctypes.sizeof(abi.CSwShard) == 64
    assert lib.jtb_struct_size(22) == ctypes.sizeof(abi.CSwResult) == 80
    assert abi.CAUSE_NAME[abi.CAUSE_NO_WITNESS] == "no-witness" and abi.CAUSE_NAME[abi.CAUSE_REAL_TIME] == "real-time"


def test_jni_shim_reports_errors_without_a_device():
    fj = _sw_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_serial_witness(0, fj.jhistory(flat(script(CONFLICT)[0])), 0, 0), np.int64)


def _sw_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_sw.c (the driver of checkSerialWitness)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_sw", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_sw.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_sw.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_sw.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_serial_witness.restype = C.c_void_p
    L.fj_check_serial_witness.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong, C.c_int]
    return fj
