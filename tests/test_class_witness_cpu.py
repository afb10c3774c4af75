"""The class witness without a GPU: CW_SEARCH against LW_SEARCH on a hand-built crowded history that only the class
pass proves (and a stale variant of it that nothing may prove), on the panel of valid bank histories (every history
LW_SEARCH proves comes back identical), on the random tiny and regrouping families (never fewer VALIDs, each one
verified), on stale and mutated histories (never VALID), the checker maps and the ABI images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, synth
from jepsen_tigerbeetle_b200 import history as H
from serial_witness import verify
from test_lifted_witness_cpu import LIFTED
from test_repaired_witness_cpu import panel
from test_serial_witness_cpu import CONFLICT, LATE, lookup_free
from test_transfer_lookups_cpu import explainable, flat, ops_idx, random_tiny, tr
from test_transfer_placement_cpu import regrouping, script


def cw(h, **kw):
    r = M.check_class_witness(h, **kw)
    verify(h, r)
    return r


def same_as_lw(lw, r):
    """r (CW_SEARCH) returns what lw (LW_SEARCH) returns, with no class pass."""
    assert {f: lw[f] for f in abi.LW_RESULT_FIELDS if not f.startswith("seconds")} == \
        {f: r[f] for f in abi.LW_RESULT_FIELDS if not f.startswith("seconds")}
    assert [{f: s[f] for f in abi.LW_SHARD_FIELDS} for s in lw["shards"]] == \
        [{f: s[f] for f in abi.LW_SHARD_FIELDS} for s in r["shards"]]
    assert all(s["class_cause"] == s["class_rounds"] == s["n_handed"] == 0 for s in r["shards"])
    assert np.array_equal(lw["commit_read"], r["commit_read"])


def crowded(n_t=220, seen=200, n_r=200, stale=False):
    """n_t :info transfers 1 -> 2 of amount 1 invoked before the first read, reads of 1, 2, .., n_r and two more of n_r,
    and a final lookup that sees the first `seen` of them.  Every gap gathers all of them, past the 128-candidate cap.
    stale: transfer seen - 1 is invoked only after the reads, so the read of n_r needs a transfer it cannot see."""
    late = {seen - 1} if stale else set()
    steps = [("t", f"x{k}", 1) for k in range(n_t) if k not in late]
    steps += [("info", f"x{k}") for k in range(n_t) if k not in late]
    steps += [("r", v) for v in range(1, n_r + 1)] + [("r", n_r), ("r", n_r)]
    steps += [("t", f"x{k}", 1) for k in late] + [("info", f"x{k}") for k in late]
    steps += [("l", [f"x{k}" for k in range(seen)])]
    return steps


CROWDED = crowded()


def test_crowded_pair():
    h = flat(script(CROWDED)[0])
    assert M.check_transfer_placement(h)["shards"][0]["valid"] == H.UNKNOWN
    lw = M.check_lifted_witness(h)["shards"][0]
    assert (lw["valid"], lw["cause"]) == (H.UNKNOWN, abi.CAUSE_UNDECIDED)
    r = cw(h)
    s = r["shards"][0]
    assert (s["valid"], s["cause"], s["class_cause"], s["class_rounds"], s["n_handed"]) == (H.VALID, 0, 0, 1, 200)
    assert (s["n_committed"], s["n_committed_crashed"], s["n_after"]) == (200, 200, 0)
    # the earliest 200 by invocation, one per read of 1..200; the 20 the lookup missed never commit
    assert (r["commit_read"][200:] == abi.SW_NEVER).all() and (r["commit_read"][:200] >= 0).all()


def test_stale_crowded_pair_is_never_valid():
    h = flat(script(crowded(stale=True))[0])
    s = cw(h)["shards"][0]
    assert s["valid"] == H.UNKNOWN and s["class_cause"] == abi.CAUSE_NO_WITNESS


# (proved by LW_SEARCH, proved by CW_SEARCH) on the panel of each size
PANEL = {10**4: (8, 8), 10**5: (7, 7)}


@pytest.mark.parametrize("ops", [10**4, 10**5])
def test_panel(ops):
    n_lw = n_cw = 0
    for key, h in panel(ops).items():
        lw = M.check_lifted_witness(h)
        r = cw(h)
        if lw["valid"] == H.VALID:
            same_as_lw(lw, r)
        n_lw += lw["valid"] == H.VALID
        n_cw += r["valid"] == H.VALID
        s = r["shards"][0]
        print(key, "LW", abi.CAUSE_NAME.get(lw["shards"][0]["cause"], "VALID"), "CW",
              abi.CAUSE_NAME.get(s["cause"], "VALID"), "class cause", abi.CAUSE_NAME.get(s["class_cause"]),
              "class rounds", s["class_rounds"], "handed", s["n_handed"])
    assert (n_lw, n_cw) == PANEL[ops]


# split_amount shows amount - 1 of a concurrent transfer; at p_info 0.02 a crashed transfer can make up the difference,
# and the class pass proves one such history (the verifier accepts the proof), so it is held to p_info 0
@pytest.mark.parametrize("variant", ["stale", "lost_transfer", "torn_transfer", "torn_pair", "split_amount"])
def test_stale_and_mutated_are_never_valid(variant):
    for seed in (1, 2):
        for p_info in (0.0,) if variant == "split_amount" else (0.0, 0.02):
            spec = synth.SynthSpec("bank", 10**4, 32, seed, n_accounts=8, final_reads=True, tau_think_ns=0.0,
                                   p_info=p_info, stale_read=variant == "stale")
            h = synth.generate_ledger_lookups(spec, **({} if variant == "stale" else {variant: True}))
            assert cw(h)["valid"] != H.VALID


@pytest.mark.parametrize("gen", ["tiny", "regrouping"])
def test_random_histories(gen, oracle_mod):
    rng = np.random.default_rng(103 if gen == "tiny" else 107)
    model = H.make_model(H.MODEL_BANK, accounts=range(1, 3))
    n_lw = n_cw = 0
    for _ in range(2000):
        ops, recs = random_tiny(rng) if gen == "tiny" else regrouping(rng)
        h = flat(ops)
        lw = M.check_lifted_witness(h)
        r = cw(h)
        n_lw += lw["valid"] == H.VALID
        if lw["valid"] == H.VALID:
            same_as_lw(lw, r)
        if r["valid"] != H.VALID:
            continue
        n_cw += 1
        assert explainable(lookup_free(recs)), ops
        bank = H.flatten_ops(ops_idx([o for o in ops if o["value"] and not any(m[0] == "l-t" for m in o["value"])]),
                             "bank")
        assert oracle_mod.check_linearizable(bank, model, oracle_mod.ALGO_WGL_COMPACT)["valid"] == H.VALID, ops
    print(f"{gen}: LW_SEARCH proves {n_lw}, CW_SEARCH {n_cw}")
    assert n_cw >= n_lw == {"tiny": 1523, "regrouping": 1066}[gen]


def test_errors():
    with pytest.raises(RuntimeError, match="negative amount"):
        M.check_class_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]))
    with pytest.raises(RuntimeError, match="reserved"):
        M.check_class_witness(flat([tr(0, "invoke", 1, 2, 1, 1)]), flags=1)


class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_class_witness(self, h, max_nodes=0, max_rounds=0, max_repairs=0, max_lifts=0, witness=False):
        return M.check_class_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, max_repairs=max_repairs,
                                     max_lifts=max_lifts, witness=witness)


def test_checker_result_map():
    c = checker.class_witness_checker(ctx=_FakeCtx())
    r = c.check({}, ops_idx(script(CROWDED)[0]))
    assert r["valid?"] is True and (r["class-rounds"], r["handed-count"], r["committed-crashed-count"]) == \
        (1, 200, 200)
    assert "class-cause" not in r and "cause" not in r
    r = c.check({}, ops_idx(script(crowded(stale=True))[0]))
    assert r["valid?"] == "unknown" and r["cause"] == "undecided" and r["class-cause"] == "no-witness"
    r = c.check({}, ops_idx(script(LIFTED)[0]))
    assert r["valid?"] is True and (r["repairs"], r["lifts"], r["class-rounds"], r["handed-count"]) == (10, 5, 0, 0)
    r = c.check({}, ops_idx(LATE))
    assert r["valid?"] == "unknown" and r["cause"] == "real-time" and r["class-cause"] == "real-time"
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, class_witness=True)
    assert "class-witness" in comp.checkers
    assert "class-witness" not in checker.ledger_checker(linear=False).checkers
    assert checker.independent_checker(checker.class_witness_checker(ctx=_FakeCtx()))._model() == "ledger-lookups"
    c = checker.class_witness_checker({"max-nodes": 7, "max-rounds": 3, "max-repairs": 4, "max-lifts": 5},
                                      ctx=_FakeCtx())
    assert (c.max_nodes, c.max_rounds, c.max_repairs, c.max_lifts) == (7, 3, 4, 5)
    r = checker.independent_checker(checker.class_witness_checker(ctx=_FakeCtx())).check(
        {}, H.concat_keys([flat(script(CROWDED)[0]), flat(script(CONFLICT)[0])]))
    assert r["valid?"] is True


def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(25) == ctypes.sizeof(abi.CLwShard) == 80
    assert lib.jtb_struct_size(26) == ctypes.sizeof(abi.CLwResult) == 112
    assert lib.jtb_struct_size(27) == ctypes.sizeof(abi.CCwShard) == 96
    assert lib.jtb_struct_size(28) == ctypes.sizeof(abi.CCwResult) == 128
    assert lib.jtb_struct_size(29) == -1
    assert lib.jtb_abi_version() == abi.ABI_VERSION == 10


def test_jni_shim_reports_errors_without_a_device():
    fj = cw_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_class_witness(0, fj.jhistory(flat(script(CONFLICT)[0])), 0, 0, 0, 0), np.int64)


def cw_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_cw.c (the driver of checkClassWitness)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_cw", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_cw.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_cw.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_cw.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_class_witness.restype = C.c_void_p
    L.fj_check_class_witness.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int]
    return fj
