"""The repaired serial witness without a GPU: RW_SEARCH against SW_SEARCH on a panel of valid bank histories (every
history SW_SEARCH proves comes back identical, and more are proved), on the random tiny and regrouping families
(never fewer VALIDs, each one verified), on stale and mutated histories (never VALID), the checker maps and the ABI
images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, synth
from jepsen_tigerbeetle_b200 import history as H
from serial_witness import verify
from test_serial_witness_cpu import CONFLICT, LATE, hand_histories, lookup_free
from test_transfer_lookups_cpu import explainable, flat, ops_idx, random_tiny, tr
from test_transfer_placement_cpu import regrouping, script


def rw(h, **kw):
    r = M.check_repaired_witness(h, **kw)
    verify(h, r)
    return r


def panel(ops):
    """The valid bank histories of one size: 8 and 64 accounts, p_info 0 and 0.02, seeds 1 and 2, τ_think 0."""
    return {(ops, n, p, seed): synth.generate_ledger_lookups(synth.SynthSpec(
        "bank", ops, 32, seed, p_info=p, n_accounts=n, final_reads=True, tau_think_ns=0.0))
        for n in (8, 64) for p in (0.0, 0.02) for seed in (1, 2)}


def same_as_sw(sw, r):
    assert {f: sw[f] for f in abi.SW_RESULT_FIELDS if not f.startswith("seconds")} == \
        {f: r[f] for f in abi.SW_RESULT_FIELDS if not f.startswith("seconds")}
    assert [{f: s[f] for f in abi.SW_SHARD_FIELDS} for s in sw["shards"]] == \
        [{f: s[f] for f in abi.SW_SHARD_FIELDS} for s in r["shards"]]
    assert all(s["repairs"] == s["n_bans"] == 0 for s in r["shards"])
    assert np.array_equal(sw["commit_read"], r["commit_read"])


# (proved by SW_SEARCH, proved by RW_SEARCH) on the panel of each size
PANEL = {10**4: (5, 8), 10**5: (3, 5)}


@pytest.mark.parametrize("ops", [10**4, 10**5])
def test_panel(ops):
    n_sw = n_rw = 0
    for key, h in panel(ops).items():
        sw = M.check_serial_witness(h)
        r = rw(h)
        if sw["valid"] == H.VALID:
            same_as_sw(sw, r)
        n_sw += sw["valid"] == H.VALID
        n_rw += r["valid"] == H.VALID
        s = r["shards"][0]
        print(key, "SW", abi.CAUSE_NAME.get(sw["shards"][0]["cause"], "VALID"), "RW",
              abi.CAUSE_NAME.get(s["cause"], "VALID"), "repairs", s["repairs"], "bans", s["n_bans"])
    assert (n_sw, n_rw) == PANEL[ops]


def test_each_repair_kind():
    """A steal proves a history SW_SEARCH leaves no-witness; real-time bans prove one it leaves real-time."""
    for ops, n, seed, cause in ((10**5, 8, 2, abi.CAUSE_NO_WITNESS), (10**4, 8, 1, abi.CAUSE_REAL_TIME)):
        h = synth.generate_ledger_lookups(synth.SynthSpec("bank", ops, 32, seed, n_accounts=n, final_reads=True,
                                                          tau_think_ns=0.0))
        assert M.check_serial_witness(h)["shards"][0]["cause"] == cause
        s = rw(h)["shards"][0]
        assert s["valid"] == H.VALID and s["repairs"] > 0 and s["n_bans"] > 0


def test_max_repairs():
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10**4, 32, 1, n_accounts=8, final_reads=True,
                                                      tau_think_ns=0.0))
    full = rw(h)
    assert full["valid"] == H.VALID and full["repairs"] == 2
    one = rw(h, max_repairs=1)
    assert one["valid"] == H.UNKNOWN and one["repairs"] == 1
    assert rw(h, max_repairs=abi.RW_DEFAULT_MAX_REPAIRS)["shards"] == full["shards"]


@pytest.mark.parametrize("variant", ["stale", "lost_transfer", "torn_transfer", "torn_pair", "split_amount"])
def test_stale_and_mutated_are_never_valid(variant):
    for seed in (1, 2):
        spec = synth.SynthSpec("bank", 10**4, 32, seed, n_accounts=8, final_reads=True, tau_think_ns=0.0,
                               stale_read=variant == "stale")
        h = synth.generate_ledger_lookups(spec, **({} if variant == "stale" else {variant: True}))
        assert rw(h)["valid"] != H.VALID


# the serial-witness check's hand cases that the repair proves: one witness round leaves the larger gap of CONFLICT
# unfixed; its steal takes {x} from the smaller gap (a ban), which then chooses {y, z}
REPAIRED = {"conflict, one round"}


def test_hand_cases():
    for name, h, kw, cause in hand_histories():
        sw = M.check_serial_witness(h, **kw)
        r = rw(h, **kw)
        if sw["valid"] == H.VALID:
            same_as_sw(sw, r)
        elif name in REPAIRED:
            s = r["shards"][0]
            assert (s["valid"], s["repairs"], s["n_bans"]) == (H.VALID, 1, 1), name
            assert r["commit_read"].tolist() == [6, 4, 4]
        else:
            assert r["shards"][0]["cause"] == cause, name


@pytest.mark.parametrize("gen", ["tiny", "regrouping"])
def test_random_histories(gen, oracle_mod):
    rng = np.random.default_rng(103 if gen == "tiny" else 107)
    model = H.make_model(H.MODEL_BANK, accounts=range(1, 3))
    n_sw = n_rw = 0
    for _ in range(2000):
        ops, recs = random_tiny(rng) if gen == "tiny" else regrouping(rng)
        h = flat(ops)
        sw = M.check_serial_witness(h)
        r = rw(h)
        n_sw += sw["valid"] == H.VALID
        if sw["valid"] == H.VALID:
            same_as_sw(sw, r)
        if r["valid"] != H.VALID:
            continue
        n_rw += 1
        assert explainable(lookup_free(recs)), ops
        bank = H.flatten_ops(ops_idx([o for o in ops if o["value"] and not any(m[0] == "l-t" for m in o["value"])]),
                             "bank")
        assert oracle_mod.check_linearizable(bank, model, oracle_mod.ALGO_WGL_COMPACT)["valid"] == H.VALID, ops
    print(f"{gen}: SW_SEARCH proves {n_sw}, RW_SEARCH {n_rw}")
    assert n_rw >= n_sw == {"tiny": 1523, "regrouping": 1066}[gen]


def test_errors():
    with pytest.raises(RuntimeError, match="negative amount"):
        M.check_repaired_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]))
    with pytest.raises(RuntimeError, match="reserved"):
        M.check_repaired_witness(flat([tr(0, "invoke", 1, 2, 1, 1)]), flags=1)


class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_repaired_witness(self, h, max_nodes=0, max_rounds=0, max_repairs=0, witness=False):
        return M.check_repaired_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, max_repairs=max_repairs,
                                        witness=witness)


def test_checker_result_map():
    c = checker.repaired_witness_checker(ctx=_FakeCtx())
    r = c.check({}, ops_idx(script(CONFLICT)[0]))
    assert r["valid?"] is True and (r["rounds"], r["repairs"], r["ban-count"]) == (2, 0, 0)
    r = c.check({}, ops_idx(LATE))
    assert r["valid?"] == "unknown" and r["cause"] == "real-time" and r["transfer-id"] == 1
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, repaired_witness=True)
    assert "repaired-witness" in comp.checkers
    assert "repaired-witness" not in checker.ledger_checker(linear=False).checkers
    assert checker.independent_checker(checker.repaired_witness_checker(ctx=_FakeCtx()))._model() == "ledger-lookups"
    c = checker.repaired_witness_checker({"max-nodes": 7, "max-rounds": 3, "max-repairs": 4}, ctx=_FakeCtx())
    assert (c.max_nodes, c.max_rounds, c.max_repairs) == (7, 3, 4)


def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(23) == ctypes.sizeof(abi.CRwShard) == 72
    assert lib.jtb_struct_size(24) == ctypes.sizeof(abi.CRwResult) == 96
    assert lib.jtb_abi_version() == abi.ABI_VERSION == 10


def test_jni_shim_reports_errors_without_a_device():
    fj = rw_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_repaired_witness(0, fj.jhistory(flat(script(CONFLICT)[0])), 0, 0, 0), np.int64)


def rw_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_rw.c (the driver of checkRepairedWitness)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_rw", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_rw.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_rw.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_rw.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_repaired_witness.restype = C.c_void_p
    L.fj_check_repaired_witness.argtypes = [C.c_longlong, C.c_void_p, C.c_longlong, C.c_int, C.c_int]
    return fj
