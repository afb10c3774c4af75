"""The lifted serial witness without a GPU: LW_SEARCH against RW_SEARCH on the panel of valid bank histories (every
history RW_SEARCH proves comes back identical, and more are proved), on the random tiny and regrouping families (never
fewer VALIDs, each one verified), on stale and mutated histories (never VALID), two small hand cases, the checker maps
and the ABI images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, synth
from jepsen_tigerbeetle_b200 import history as H
from serial_witness import verify
from test_repaired_witness_cpu import panel
from test_serial_witness_cpu import CONFLICT, LATE, lookup_free
from test_transfer_lookups_cpu import explainable, flat, ops_idx, random_tiny, tr
from test_transfer_placement_cpu import regrouping, script


def lw(h, **kw):
    r = M.check_lifted_witness(h, **kw)
    verify(h, r)
    return r


def same_as_rw(rw, r):
    """r (LW_SEARCH) returns what rw (RW_SEARCH) returns, with no lift step."""
    assert {f: rw[f] for f in abi.RW_RESULT_FIELDS if not f.startswith("seconds")} == \
        {f: r[f] for f in abi.RW_RESULT_FIELDS if not f.startswith("seconds")}
    assert [{f: s[f] for f in abi.RW_SHARD_FIELDS} for s in rw["shards"]] == \
        [{f: s[f] for f in abi.RW_SHARD_FIELDS} for s in r["shards"]]
    assert all(s["lifts"] == s["n_lifted"] == 0 for s in r["shards"])
    assert np.array_equal(rw["commit_read"], r["commit_read"])


# (proved by RW_SEARCH, proved by LW_SEARCH) on the panel of each size
PANEL = {10**4: (8, 8), 10**5: (5, 7)}


@pytest.mark.parametrize("ops", [10**4, 10**5])
def test_panel(ops):
    n_rw = n_lw = 0
    for key, h in panel(ops).items():
        rw = M.check_repaired_witness(h)
        r = lw(h)
        if rw["valid"] == H.VALID:
            same_as_rw(rw, r)
        n_rw += rw["valid"] == H.VALID
        n_lw += r["valid"] == H.VALID
        s = r["shards"][0]
        print(key, "RW", abi.CAUSE_NAME.get(rw["shards"][0]["cause"], "VALID"), "LW",
              abi.CAUSE_NAME.get(s["cause"], "VALID"), "repairs", s["repairs"], "lifts", s["lifts"], "lifted",
              s["n_lifted"], "bans", s["n_bans"])
    assert (n_rw, n_lw) == PANEL[ops]


# a crashed a = 3 and :ok b..f; reads of 4 and 12.  K14's repairs leave a gap with every candidate banned; lift steps
# give the bans back and the witness is found
LIFTED = [("t", "a", 3), ("t", "b", 2), ("t", "c", 3), ("t", "d", 1), ("t", "e", 2), ("r", 4), ("t", "f", 2),
          ("r", 12), ("info", "a"), ("ok", "b"), ("ok", "c"), ("ok", "d"), ("ok", "e"), ("ok", "f")]
# reads of 2 and 6 with 5 invoked before the second: no witness exists; lift steps run, each pair lifts once, and the
# shard ends UNKNOWN within its bounds
CYCLING = [("t", "a", 1), ("t", "b", 2), ("t", "c", 1), ("t", "d", 1), ("r", 2), ("r", 6), ("t", "e", 1),
           ("t", "f", 2), ("info", "a"), ("info", "b"), ("ok", "c"), ("ok", "d"), ("info", "e"), ("ok", "f")]


def test_hand_lift():
    h = flat(script(LIFTED)[0])
    rs = M.check_repaired_witness(h)["shards"][0]
    assert (rs["valid"], rs["cause"], rs["repairs"], rs["n_bans"]) == (H.UNKNOWN, abi.CAUSE_NO_WITNESS, 4, 5)
    r = lw(h)
    s = r["shards"][0]
    assert (s["valid"], s["repairs"], s["n_bans"], s["lifts"], s["n_lifted"]) == (H.VALID, 10, 11, 5, 8)
    assert explainable(lookup_free(script(LIFTED)[1]))
    one = lw(h, max_lifts=1)["shards"][0]
    assert one["valid"] == H.UNKNOWN and one["lifts"] == 1
    # out of max_repairs, K14's verdict stands and no lift step runs
    short = lw(h, max_repairs=1)
    same_as_rw(M.check_repaired_witness(h, max_repairs=1), short)


def test_hand_cycle_ends_within_bounds():
    h = flat(script(CYCLING)[0])
    s = lw(h)["shards"][0]
    assert (s["valid"], s["cause"], s["lifts"], s["n_lifted"]) == (H.UNKNOWN, abi.CAUSE_NO_WITNESS, 2, 4)
    assert s["repairs"] <= abi.RW_DEFAULT_MAX_REPAIRS + abi.LW_DEFAULT_MAX_LIFTS
    assert not explainable(lookup_free(script(CYCLING)[1]))


@pytest.mark.parametrize("variant", ["stale", "lost_transfer", "torn_transfer", "torn_pair", "split_amount"])
def test_stale_and_mutated_are_never_valid(variant):
    for seed in (1, 2):
        spec = synth.SynthSpec("bank", 10**4, 32, seed, n_accounts=8, final_reads=True, tau_think_ns=0.0,
                               stale_read=variant == "stale")
        h = synth.generate_ledger_lookups(spec, **({} if variant == "stale" else {variant: True}))
        assert lw(h)["valid"] != H.VALID


@pytest.mark.parametrize("gen", ["tiny", "regrouping"])
def test_random_histories(gen, oracle_mod):
    rng = np.random.default_rng(103 if gen == "tiny" else 107)
    model = H.make_model(H.MODEL_BANK, accounts=range(1, 3))
    n_rw = n_lw = 0
    for _ in range(2000):
        ops, recs = random_tiny(rng) if gen == "tiny" else regrouping(rng)
        h = flat(ops)
        rw = M.check_repaired_witness(h)
        r = lw(h)
        n_rw += rw["valid"] == H.VALID
        if rw["valid"] == H.VALID:
            same_as_rw(rw, r)
        if r["valid"] != H.VALID:
            continue
        n_lw += 1
        assert explainable(lookup_free(recs)), ops
        bank = H.flatten_ops(ops_idx([o for o in ops if o["value"] and not any(m[0] == "l-t" for m in o["value"])]),
                             "bank")
        assert oracle_mod.check_linearizable(bank, model, oracle_mod.ALGO_WGL_COMPACT)["valid"] == H.VALID, ops
    print(f"{gen}: RW_SEARCH proves {n_rw}, LW_SEARCH {n_lw}")
    assert n_lw >= n_rw == {"tiny": 1523, "regrouping": 1066}[gen]


def test_errors():
    with pytest.raises(RuntimeError, match="negative amount"):
        M.check_lifted_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]))
    with pytest.raises(RuntimeError, match="reserved"):
        M.check_lifted_witness(flat([tr(0, "invoke", 1, 2, 1, 1)]), flags=1)


class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_lifted_witness(self, h, max_nodes=0, max_rounds=0, max_repairs=0, max_lifts=0, witness=False):
        return M.check_lifted_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, max_repairs=max_repairs,
                                      max_lifts=max_lifts, witness=witness)


def test_checker_result_map():
    c = checker.lifted_witness_checker(ctx=_FakeCtx())
    r = c.check({}, ops_idx(script(CONFLICT)[0]))
    assert r["valid?"] is True and (r["rounds"], r["repairs"], r["ban-count"], r["lifts"], r["lifted-count"]) == \
        (2, 0, 0, 0, 0)
    r = c.check({}, ops_idx(script(LIFTED)[0]))
    assert r["valid?"] is True and (r["repairs"], r["lifts"], r["lifted-count"]) == (10, 5, 8)
    r = c.check({}, ops_idx(LATE))
    assert r["valid?"] == "unknown" and r["cause"] == "real-time" and r["transfer-id"] == 1
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, lifted_witness=True)
    assert "lifted-witness" in comp.checkers
    assert "lifted-witness" not in checker.ledger_checker(linear=False).checkers
    assert checker.independent_checker(checker.lifted_witness_checker(ctx=_FakeCtx()))._model() == "ledger-lookups"
    c = checker.lifted_witness_checker({"max-nodes": 7, "max-rounds": 3, "max-repairs": 4, "max-lifts": 5},
                                       ctx=_FakeCtx())
    assert (c.max_nodes, c.max_rounds, c.max_repairs, c.max_lifts) == (7, 3, 4, 5)


def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(23) == ctypes.sizeof(abi.CRwShard) == 72
    assert lib.jtb_struct_size(24) == ctypes.sizeof(abi.CRwResult) == 96
    assert lib.jtb_struct_size(25) == ctypes.sizeof(abi.CLwShard) == 80
    assert lib.jtb_struct_size(26) == ctypes.sizeof(abi.CLwResult) == 112
    assert lib.jtb_abi_version() == abi.ABI_VERSION == 10


def test_jni_shim_reports_errors_without_a_device():
    fj = lw_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_lifted_witness(0, fj.jhistory(flat(script(CONFLICT)[0])), 0, 0, 0, 0), np.int64)


def lw_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_lw.c (the driver of checkLiftedWitness)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_lw", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_lw.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_lw.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_lw.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_lifted_witness.restype = C.c_void_p
    L.fj_check_lifted_witness.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int]
    return fj
