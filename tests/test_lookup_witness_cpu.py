"""The lookup witness without a GPU: LK_SEARCH against LK_BRUTE (the definition) and the independent verifier on the
random tiny and regrouping families with lookups, LK_SEARCH equal to CW_SEARCH on lookup-free histories, hand cases
for a final lookup of crashed transfers, two crossing lookups and a mid-run lookup that returns a crashed transfer the
witness commits only in a later gap, the search for histories K9 and K16 pass and LK_BRUTE rejects, the checker maps,
the ABI images of the new structs and the JNI shim."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker
from jepsen_tigerbeetle_b200 import history as H
from lookup_witness import verify
from test_class_witness_cpu import CROWDED
from test_monotonic_cpu import inv_r, rd
from test_transfer_lookups_cpu import flat, inv_l, lk as lk_op, ops_idx, random_tiny, tr
from test_transfer_placement_cpu import script


def lk(h, **kw):
    r = M.check_lookup_witness(h, **kw)
    verify(h, r)
    return r


def same_as_cw(cw, r):
    """r (LK_SEARCH) returns what cw (CW_SEARCH) returns, with no lookup placed."""
    assert {f: cw[f] for f in abi.CW_RESULT_FIELDS if not f.startswith("seconds")} == \
        {f: r[f] for f in abi.CW_RESULT_FIELDS if not f.startswith("seconds")}
    assert [{f: s[f] for f in abi.CW_SHARD_FIELDS} for s in cw["shards"]] == \
        [{f: s[f] for f in abi.CW_SHARD_FIELDS} for s in r["shards"]]
    assert all(s["lookup_cause"] == s["n_lookups_placed"] == 0 and s["lookup_fail_index"] == -1 for s in r["shards"])
    assert np.array_equal(cw["commit_read"], r["commit_read"])


def regrouping_lookups(rng):
    """test_transfer_placement_cpu's regrouping family with lookups: after a read, half the time, a lookup that
    returns a random subset of the transfers invoked so far, and a final lookup of another such subset."""
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
            if rng.random() < 0.5:
                steps.append(("l", [t[1] for t in invoked if rng.random() < 0.6]))
    steps += [(str(rng.choice(["ok", "info"])), name) for name in open_]
    steps.append(("l", [t[1] for t in invoked if rng.random() < 0.8]))
    return script(steps)


@pytest.mark.parametrize("gen", ["tiny", "regrouping"])
def test_random_histories(gen):
    rng = np.random.default_rng(109 if gen == "tiny" else 113)
    n_brute = n_lk = n_cw = n_placed = n_k16_only = 0
    for _ in range(2000):
        ops, _ = random_tiny(rng) if gen == "tiny" else regrouping_lookups(rng)
        h = flat(ops)
        cw = M.check_class_witness(h)
        r = lk(h)
        brute = M.check_lookup_witness(h, algo=M.LK_BRUTE)["valid"] == H.VALID
        n_brute += brute
        n_cw += cw["valid"] == H.VALID
        if r["valid"] == H.VALID:
            assert brute, ops
            n_lk += 1
            n_placed += r["n_lookups_placed"] > 0
        if abi.n_ok_lookups(h) == 0:
            same_as_cw(cw, r)
        if cw["valid"] == H.VALID and not brute:   # K16 proves it, no serial order with lookups exists: K9 catches it
            n_k16_only += 1
            assert M.check_transfer_lookups(h, M.TL_SWEEP)["valid"] != H.VALID, ops
    print(f"{gen}: LK_BRUTE serializable {n_brute}, LK_SEARCH proves {n_lk} ({n_placed} with lookups placed), "
          f"CW_SEARCH {n_cw}, of which {n_k16_only} have no serial order with their lookups (K9 flags each)")
    assert n_lk == {"tiny": 1005, "regrouping": 563}[gen] and n_lk <= n_brute


def test_lookup_free_equals_class_witness():
    rng = np.random.default_rng(127)
    for _ in range(500):
        ops, _ = random_tiny(rng)
        ops = [o for o in ops if o["value"] and not any(m[0] == "l-t" for m in o["value"])]
        h = flat(ops)
        same_as_cw(M.check_class_witness(h), lk(h))
    h = flat(script(CROWDED[:-1])[0])
    same_as_cw(M.check_class_witness(h), lk(h))


def test_final_lookup_of_crashed_transfers():
    """The crowded pair: the class witness commits 200 of 220 :info transfers and leaves 20 uncommitted; a final lookup
    that shows 210 commits the 10 more after the last read."""
    steps = CROWDED[:-1] + [("l", [f"x{k}" for k in range(210)])]
    h = flat(script(steps)[0])
    r = lk(h)
    s = r["shards"][0]
    assert (s["valid"], s["lookup_cause"], s["n_lookups_placed"]) == (H.VALID, 0, 1)
    assert (r["commit_read"][200:210] == abi.SW_AFTER).all() and (r["commit_read"][210:] == abi.SW_NEVER).all()
    assert list(r["lookup_read"]) == [abi.SW_AFTER]
    assert (M.check_class_witness(h)["commit_read"][200:] == abi.SW_NEVER).all()


# two :info transfers a, b before the reads 0 and 2 (both commit in gap 1), and between the reads two lookups
# concurrent with everything, one showing a and the other b: their sets cross
CROSSING = [("t", "a", 1), ("t", "b", 1), ("info", "a"), ("info", "b"), ("r", 0), ("l", ["a"]), ("l", ["b"]),
            ("r", 2)]
def test_crossing_lookups():
    ops = script(CROSSING)[0]
    h = flat(ops)
    cw = M.check_class_witness(h)
    assert cw["valid"] == H.VALID
    r = lk(h)
    s = r["shards"][0]
    assert (s["valid"], s["cause"], s["lookup_cause"]) == (H.UNKNOWN, abi.CAUSE_LOOKUP, abi.CAUSE_LOOKUP)
    assert s["lookup_fail_index"] == s["fail_index"] >= 0 and s["n_lookups_placed"] == 0
    assert (r["commit_read"] == abi.SW_NEVER).all() and (r["lookup_read"] == abi.SW_NEVER).all()
    assert M.check_lookup_witness(h, algo=M.LK_BRUTE)["valid"] == H.INVALID


# a mid-run lookup that returns a crashed transfer the witness commits only in a later gap: :info c and :ok d of amount
# 1 from account 1 to 2; the lookup is invoked before d completes and completes after the first read is invoked, so K9
# needs neither d in it nor c in the first read; d completes before the first read (1), so the witness puts d in gap 0
# and c in gap 1 (the second read, 2).  The lookup returns c (gap 1) and lacks d (gap 0): lo > hi.  There is no serial
# order: c before the lookup before d before the first read before c.  K9 and K16 pass it.
EARLY = [tr(1, "invoke", 1, 2, 1, 1), tr(2, "invoke", 1, 2, 1, 2), inv_l(3), tr(2, "ok", 1, 2, 1, 2), inv_r(4, [1, 2]),
         lk_op(3, [(1, 1, 2, 1)]), rd(4, {1: (1, 0), 2: (0, 1)}), inv_r(4, [1, 2]), rd(4, {1: (2, 0), 2: (0, 2)}),
         tr(1, "info", 1, 2, 1, 1)]


def test_early_lookup():
    h = flat(EARLY)
    assert M.check_transfer_lookups(h, M.TL_SWEEP)["valid"] == H.VALID
    cw = M.check_class_witness(h)
    assert cw["valid"] == H.VALID and list(cw["commit_read"]) == [8, 6]   # c at the second read, d at the first
    r = lk(h)
    s = r["shards"][0]
    assert (s["valid"], s["cause"], s["lookup_cause"], s["lookup_fail_index"]) == \
        (H.UNKNOWN, abi.CAUSE_LOOKUP, abi.CAUSE_LOOKUP, 5)
    assert M.check_lookup_witness(h, algo=M.LK_BRUTE)["valid"] == H.INVALID


def test_errors():
    with pytest.raises(RuntimeError, match="negative amount"):
        M.check_lookup_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]))
    with pytest.raises(RuntimeError, match="reserved"):
        M.check_lookup_witness(flat([tr(0, "invoke", 1, 2, 1, 1)]), flags=1)


class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_lookup_witness(self, h, max_nodes=0, max_rounds=0, max_repairs=0, max_lifts=0, witness=False):
        return M.check_lookup_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, max_repairs=max_repairs,
                                      max_lifts=max_lifts, witness=witness)


def test_checker_result_map():
    c = checker.lookup_witness_checker(ctx=_FakeCtx())
    r = c.check({}, ops_idx(script(CROWDED)[0]))
    assert r["valid?"] is True and (r["lookups-placed-count"], r["handed-count"]) == (1, 200)
    assert "lookup-cause" not in r and "cause" not in r
    r = c.check({}, ops_idx(script(CROSSING)[0]))
    assert r["valid?"] == "unknown" and r["cause"] == r["lookup-cause"] == "lookup" and r["lookup-op"]["index"] >= 0
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, lookup_witness=True)
    assert "lookup-witness" in comp.checkers
    assert "lookup-witness" not in checker.ledger_checker(linear=False).checkers
    c = checker.lookup_witness_checker({"max-nodes": 7, "max-rounds": 3, "max-repairs": 4, "max-lifts": 5},
                                       ctx=_FakeCtx())
    assert (c.max_nodes, c.max_rounds, c.max_repairs, c.max_lifts) == (7, 3, 4, 5)


def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(29) == -1
    assert lib.jtb_struct_size(30) == ctypes.sizeof(abi.CLkShard) == 112
    assert lib.jtb_struct_size(31) == ctypes.sizeof(abi.CLkResult) == 136
    assert lib.jtb_struct_size(32) == -1


def test_jni_shim_reports_errors_without_a_device():
    fj = lk_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_lookup_witness(0, fj.jhistory(flat(script(CROSSING)[0])), 0, 0, 0, 0), np.int64)


def lk_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_lk.c (the driver of checkLookupWitness)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_lk", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_lk.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_lk.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_lk.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_lookup_witness.restype = C.c_void_p
    L.fj_check_lookup_witness.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int]
    return fj
