"""The serial-witness check on the GPU (K13) against SW_SEARCH, field by field and commit_read entry for entry, with
every VALID proof re-checked by the independent verifier (tests/serial_witness.py); C3-size, crashed, mid-history
lookup, 64-account, multi-shard and 10^6-op histories; the cross-check against the bank model's :linear; every error
path."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from serial_witness import verify
from test_monotonic_cpu import inv_r, rd
from test_read_gaps_cpu import _ones
from test_serial_witness_cpu import CONFLICT, CONFLICT_LOST, _sw_fakejvm, hand_histories
from test_transfer_lookups_cpu import flat, inv_l, lk, random_tiny, tr
from test_transfer_placement_cpu import regrouping, script

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes",
          "rounds", "shards")
MUTATIONS = ("torn_transfer", "torn_pair", "split_amount")


def agree(ctx, h, max_nodes=0, max_rounds=0):
    g = ctx.check_serial_witness(h, max_nodes, max_rounds, witness=True)
    o = M.check_serial_witness(h, max_nodes=max_nodes, max_rounds=max_rounds)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    assert np.array_equal(g["commit_read"], o["commit_read"])
    verify(h, g)
    return g


def causes(r):
    return sorted({s["cause"] for s in r["shards"]})


def test_random_tiny_histories(gpu_ctx):
    rng = np.random.default_rng(101)
    seen = set()
    for i in range(300):
        r = agree(gpu_ctx, flat(random_tiny(rng)[0]), max_nodes=(0, 1, 3)[i % 3], max_rounds=(0, 1, 2)[i % 3 - 1])
        seen.update(causes(r))
        seen.update(causes(agree(gpu_ctx, flat(regrouping(rng)[0]))))
    assert {0, abi.CAUSE_ANOMALY, abi.CAUSE_REAL_TIME} <= seen, seen


def test_hand_cases(gpu_ctx):
    for name, h, kw, cause in hand_histories():
        r = agree(gpu_ctx, h, **kw)
        assert r["shards"][0]["cause"] == cause, name
    for mr in (1, 2, 3):
        agree(gpu_ctx, flat(script(CONFLICT_LOST)[0]), max_rounds=mr)
    for n, shows in ((40, (20, 20)), (70, (35, 35)), (130, (65, 65))):
        agree(gpu_ctx, flat(_ones(n, shows)))


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("variant", ("valid", "stale", "lost_transfer") + MUTATIONS)
def test_c3_size_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, final_reads=True, stale_read=variant == "stale")
    h = synth.generate_ledger_lookups(spec, **({variant: True} if variant in MUTATIONS + ("lost_transfer",) else {}))
    g = agree(gpu_ctx, h)
    if variant != "valid":
        assert g["valid"] != H.VALID, variant
    print(variant, seed, causes(g), g["rounds"], g["n_committed_crashed"])


def test_crashed_transfers(gpu_ctx):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True))
    g = agree(gpu_ctx, h)
    print("C3 p_info 0.02:", g["valid"], causes(g), g["rounds"], g["n_committed_crashed"])


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
    muts = {2: "torn_transfer", 5: "split_amount", 6: "torn_pair"}
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05,
                                                           final_reads=True), **({muts[s]: True} if s in muts else {}))
             for s in range(1, 9)]
    parts += [h for _, h, kw, _ in hand_histories() if not kw]
    g = agree(gpu_ctx, H.concat_keys(parts))
    assert len(g["shards"]) == len(parts)


def test_million_op_history(gpu_ctx):
    """The oracle is slow here: the device result alone, re-checked by the vectorised verifier."""
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 1_000_000, 32, 1, p_info=0.02, final_reads=True))
    g = gpu_ctx.check_serial_witness(h, witness=True)
    assert g["n_reads"] > 400_000
    verify(h, g)
    print("10^6 ops, 8 accounts, p_info 0.02:", g["valid"], causes(g), g["rounds"], g["n_committed_crashed"],
          g["seconds_kernel"])


def test_linear_cross_check(gpu_ctx, oracle_mod):
    """synth.generate(spec) is the bank form of the events generate_ledger_lookups(spec) flattens: wherever the
    device's :linear search decides the bank form, a witness VALID never meets INVALID; where the CPU lazy-bank search
    has a verdict, the two agree."""
    m = H.make_model(H.MODEL_BANK, accounts=range(1, 9))
    tally = {}
    for seed in range(1, 7):
        for p_info in (0.0, 0.02):
            for stale in (False, True):
                spec = synth.SynthSpec("bank", 600, 8, seed, p_info=p_info, stale_read=stale, tau_think_ns=5e6)
                w = agree(gpu_ctx, synth.generate_ledger_lookups(spec))["valid"]
                bank = synth.generate(spec)
                lin = gpu_ctx.check_linearizable(bank, m)["valid"]
                if w == H.VALID:
                    assert lin != H.INVALID, (seed, p_info, stale)
                    o = oracle_mod.check_linearizable(bank, m, oracle_mod.ALGO_LAZY_BANK, max_configs=2_000_000)
                    assert o["valid"] != H.INVALID, (seed, p_info, stale)
                key = (p_info, lin, w)
                tally[key] = tally.get(key, 0) + 1
    print("(p_info, :linear, witness): count", tally)


def test_errors_leave_the_context_usable(gpu_ctx):
    ok = [tr(0, "invoke", 1, 2, 1, 1), tr(0, "ok", 1, 2, 1, 1)]
    good = flat(script(CONFLICT)[0])

    def raises(ops, match, mutate=None):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(NativeError, match=match):
            gpu_ctx.check_serial_witness(h, witness=True)
        assert agree(gpu_ctx, good)["valid"] == H.VALID

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", -1, 2, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, 0))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises(ok + [inv_l(1), lk(1, [(1, 1, 2, 1)])], "multiple of 5", lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "multiple of 3", lambda h: h.payload_len.__setitem__(1, 5))
    ch = H.as_c_history(flat(ok))
    shards, res = (abi.CSwShard * 1)(), abi.CSwResult()
    L = native.lib()
    assert L.jtb_check_serial_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 1, None, C.addressof(shards),
                                      C.addressof(res)) < 0
    assert "reserved" in gpu_ctx._err()
    assert L.jtb_check_serial_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 0, None, None, C.addressof(res)) < 0
    assert "null" in gpu_ctx._err()
    assert agree(gpu_ctx, good)["valid"] == H.VALID
    assert gpu_ctx.check_serial_witness(good)["shards"] == agree(gpu_ctx, good)["shards"]   # without commit_read


def test_checker_result_map(gpu_ctx):
    from jepsen_tigerbeetle_b200 import checker
    r = checker.serial_witness_checker(ctx=gpu_ctx).check({}, [dict(o, index=i) for i, o in
                                                               enumerate(script(CONFLICT)[0])])
    assert r["valid?"] is True and r["rounds"] == 2
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 600, 8, s, tau_think_ns=5e6, final_reads=True))
             for s in (1, 2, 3)]
    r = checker.independent_checker(checker.serial_witness_checker(ctx=gpu_ctx)).check({}, H.concat_keys(parts))
    assert r["valid?"] in (True, "unknown")


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkSerialWitness through the JNI shim and a fake JNIEnv returns what ctypes returns."""
    fj = _sw_fakejvm()
    handle = fj.create()
    try:
        parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, final_reads=True),
                                               torn_pair=s == 2) for s in (1, 2, 3)]
        parts += [h for _, h, kw, _ in hand_histories() if not kw]
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_serial_witness(handle, fj.jhistory(h), 0, 0), np.int64)
        g = gpu_ctx.check_serial_witness(h)
        assert v[:9].tolist() == [g[k] for k in ("valid", "n_failures", "n_reads", "n_transfers", "n_committed",
                                                 "n_committed_crashed", "n_after", "nodes", "rounds")]
        assert v[11] == h.n_shards
        for s, q in enumerate(g["shards"]):
            assert v[12 + 11 * s: 23 + 11 * s].tolist() == [q[f] for f in abi.SW_SHARD_FIELDS]
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_serial_witness(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])),
                                                        0, 0), np.int64)
    finally:
        fj.lib().fj_destroy(handle)
