"""The repaired serial witness on the GPU (K14) against RW_SEARCH, field by field and commit_read entry for entry, with
every VALID proof re-checked by the independent verifier: the panel of valid bank histories, C3 valid and mutated,
crashed, mid-history lookup, 64-account and multi-shard histories, one history per repair kind, the error paths and
the JNI shim."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from serial_witness import verify
from test_repaired_witness_cpu import REPAIRED, panel, rw_fakejvm
from test_serial_witness_cpu import CONFLICT, hand_histories
from test_transfer_lookups_cpu import flat, random_tiny, tr
from test_transfer_placement_cpu import regrouping, script

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes",
          "rounds", "repairs", "n_bans", "shards")
MUTATIONS = ("torn_transfer", "torn_pair", "split_amount")


def agree(ctx, h, max_nodes=0, max_rounds=0, max_repairs=0):
    g = ctx.check_repaired_witness(h, max_nodes, max_rounds, max_repairs, witness=True)
    o = M.check_repaired_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, max_repairs=max_repairs)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    assert np.array_equal(g["commit_read"], o["commit_read"])
    verify(h, g)
    return g


@pytest.mark.parametrize("ops", [10**4, 10**5])
def test_panel(gpu_ctx, ops):
    for key, h in panel(ops).items():
        g = agree(gpu_ctx, h)
        s = g["shards"][0]
        print(key, abi.CAUSE_NAME.get(s["cause"], "VALID"), "repairs", s["repairs"], "bans", s["n_bans"])


def test_repair_kinds_and_budgets(gpu_ctx):
    for ops, n, seed in ((10**5, 8, 2), (10**4, 8, 1)):
        h = synth.generate_ledger_lookups(synth.SynthSpec("bank", ops, 32, seed, n_accounts=n, final_reads=True,
                                                          tau_think_ns=0.0))
        assert agree(gpu_ctx, h)["valid"] == H.VALID
        for mr in (1, 2):
            agree(gpu_ctx, h, max_repairs=mr)
        agree(gpu_ctx, h, max_rounds=1)
        agree(gpu_ctx, h, max_nodes=3)


def test_hand_cases(gpu_ctx):
    for name, h, kw, cause in hand_histories():
        r = agree(gpu_ctx, h, **kw)
        assert (r["valid"] == H.VALID) if name in REPAIRED else r["shards"][0]["cause"] == cause, name


def test_random_histories(gpu_ctx):
    rng = np.random.default_rng(109)
    for i in range(200):
        agree(gpu_ctx, flat(random_tiny(rng)[0]), max_nodes=(0, 1, 3)[i % 3], max_rounds=(0, 1, 2)[i % 3 - 1])
        agree(gpu_ctx, flat(regrouping(rng)[0]), max_repairs=(0, 1)[i % 2])


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("variant", ("valid", "stale", "lost_transfer") + MUTATIONS)
def test_c3_size_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, final_reads=True, stale_read=variant == "stale")
    h = synth.generate_ledger_lookups(spec, **({variant: True} if variant in MUTATIONS + ("lost_transfer",) else {}))
    g = agree(gpu_ctx, h)
    if variant != "valid":
        assert g["valid"] != H.VALID, variant


def test_crashed_transfers(gpu_ctx):
    for seed in (1, 2):
        agree(gpu_ctx, synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, seed, p_info=0.02,
                                                                     final_reads=True)))


def test_mid_history_lookups(gpu_ctx):
    spec = synth.SynthSpec("bank", 600, 8, 2, p_info=0.05, final_reads=True)
    for kw in ({}, {"lost_transfer": True}, {"torn_pair": True}):
        agree(gpu_ctx, synth.generate_ledger_lookups(spec, p_lookup=0.05, **kw))


@pytest.mark.parametrize("kw", [{}, {"torn_pair": True}])
def test_64_accounts(gpu_ctx, kw):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, p_info=0.02,
                                                      final_reads=True), **kw)
    agree(gpu_ctx, h)


def test_multi_shard(gpu_ctx):
    """Shards that repair next to shards that stop, fail or are proved at once."""
    muts = {2: "torn_transfer", 5: "split_amount", 6: "torn_pair"}
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05,
                                                           final_reads=True), **({muts[s]: True} if s in muts else {}))
             for s in range(1, 9)]
    parts += [synth.generate_ledger_lookups(synth.SynthSpec("bank", 10**4, 32, s, n_accounts=8, final_reads=True,
                                                            tau_think_ns=0.0)) for s in (1, 2)]
    parts += [h for _, h, kw, _ in hand_histories() if not kw]
    for mr in (0, 1):
        g = agree(gpu_ctx, H.concat_keys(parts), max_repairs=mr)
        assert len(g["shards"]) == len(parts)


def test_errors_leave_the_context_usable(gpu_ctx):
    good = flat(script(CONFLICT)[0])
    with pytest.raises(NativeError, match="negative amount"):
        gpu_ctx.check_repaired_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]), witness=True)
    assert agree(gpu_ctx, good)["valid"] == H.VALID
    with pytest.raises(NativeError, match="reserved"):
        gpu_ctx.check_repaired_witness(good, flags=1)
    ch = H.as_c_history(good)
    res = abi.CRwResult()
    assert native.lib().jtb_check_repaired_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 0, 0, None, None,
                                                   C.addressof(res)) < 0
    assert "null" in gpu_ctx._err()
    assert agree(gpu_ctx, good)["valid"] == H.VALID
    assert gpu_ctx.check_repaired_witness(good)["shards"] == agree(gpu_ctx, good)["shards"]   # without commit_read


def test_checker_result_map(gpu_ctx):
    from jepsen_tigerbeetle_b200 import checker
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 10**4, 32, s, n_accounts=8, final_reads=True,
                                                           tau_think_ns=0.0)) for s in (1, 2)]
    r = checker.independent_checker(checker.repaired_witness_checker(ctx=gpu_ctx)).check({}, H.concat_keys(parts))
    assert r["valid?"] is True


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkRepairedWitness through the JNI shim and a fake JNIEnv returns what ctypes returns."""
    fj = rw_fakejvm()
    handle = fj.create()
    try:
        parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 10**4, 32, s, n_accounts=8, final_reads=True,
                                                               tau_think_ns=0.0), torn_pair=s == 3) for s in (1, 2, 3)]
        parts += [h for _, h, kw, _ in hand_histories() if not kw]
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_repaired_witness(handle, fj.jhistory(h), 0, 0, 0), np.int64)
        g = gpu_ctx.check_repaired_witness(h)
        assert v[:11].tolist() == [g[k] for k in abi.RW_RESULT_FIELDS[:11]]
        assert v[13] == h.n_shards
        for s, q in enumerate(g["shards"]):
            assert v[14 + 13 * s: 27 + 13 * s].tolist() == [q[f] for f in abi.RW_SHARD_FIELDS]
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_repaired_witness(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])),
                                                          0, 0, 0), np.int64)
    finally:
        fj.lib().fj_destroy(handle)
