"""The class witness on the GPU (K16) against CW_SEARCH, field by field and commit_read entry for entry, with every
VALID proof re-checked by the independent verifier: the crowded hand case and its stale variant, the panel of valid
bank histories, the random families, a multi-shard history, the budgets, the error paths and the JNI shim; and K15's
device results on the same inputs, which must stay as LW_SEARCH computes them."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from serial_witness import verify
from test_class_witness_cpu import CROWDED, crowded, cw_fakejvm
from test_lifted_witness_cpu import CYCLING, LIFTED
from test_repaired_witness_cpu import panel
from test_serial_witness_cpu import CONFLICT, hand_histories
from test_transfer_lookups_cpu import flat, random_tiny, tr
from test_transfer_placement_cpu import regrouping, script

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes",
          "rounds", "repairs", "n_bans", "lifts", "n_lifted", "class_rounds", "n_handed", "shards")
LW_FIELDS = FIELDS[:13] + ("shards",)


def agree(ctx, h, max_nodes=0, max_rounds=0, max_repairs=0, max_lifts=0):
    g = ctx.check_class_witness(h, max_nodes, max_rounds, max_repairs, max_lifts, witness=True)
    o = M.check_class_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, max_repairs=max_repairs,
                              max_lifts=max_lifts)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    assert np.array_equal(g["commit_read"], o["commit_read"])
    verify(h, g)
    return g


def agree_lw(ctx, h, **kw):
    g = ctx.check_lifted_witness(h, witness=True, **kw)
    o = M.check_lifted_witness(h, **kw)
    assert {k: g[k] for k in LW_FIELDS} == {k: o[k] for k in LW_FIELDS}
    assert np.array_equal(g["commit_read"], o["commit_read"])
    return g


def test_crowded_pair(gpu_ctx):
    h = flat(script(CROWDED)[0])
    assert agree_lw(gpu_ctx, h)["shards"][0]["cause"] == abi.CAUSE_UNDECIDED
    s = agree(gpu_ctx, h)["shards"][0]
    assert (s["valid"], s["class_rounds"], s["n_handed"]) == (H.VALID, 1, 200)
    for kw in ({"max_rounds": 1}, {"max_nodes": 1}, {"max_repairs": 1, "max_lifts": 1}):
        agree(gpu_ctx, h, **kw)
    stale = flat(script(crowded(stale=True))[0])
    s = agree(gpu_ctx, stale)["shards"][0]
    assert s["valid"] == H.UNKNOWN and s["class_cause"] == abi.CAUSE_NO_WITNESS
    agree_lw(gpu_ctx, stale)


@pytest.mark.parametrize("ops", [10**4, 10**5])
def test_panel(gpu_ctx, ops):
    for key, h in panel(ops).items():
        g = agree(gpu_ctx, h)
        agree_lw(gpu_ctx, h)
        s = g["shards"][0]
        print(key, abi.CAUSE_NAME.get(s["cause"], "VALID"), "class cause", abi.CAUSE_NAME.get(s["class_cause"]),
              "class rounds", s["class_rounds"], "handed", s["n_handed"])


def test_hand_cases(gpu_ctx):
    for steps in (LIFTED, CYCLING, crowded(n_t=6, seen=5, n_r=5), crowded(n_t=6, seen=5, n_r=5, stale=True)):
        h = flat(script(steps)[0])
        agree(gpu_ctx, h)
        agree(gpu_ctx, h, max_rounds=1)
    for name, h, kw, cause in hand_histories():
        agree(gpu_ctx, h, **kw)


def test_random_histories(gpu_ctx):
    rng = np.random.default_rng(127)
    for i in range(200):
        agree(gpu_ctx, flat(random_tiny(rng)[0]), max_nodes=(0, 1, 3)[i % 3], max_rounds=(0, 1, 2)[i % 3 - 1])
        agree(gpu_ctx, flat(regrouping(rng)[0]), max_repairs=(0, 1)[i % 2], max_lifts=(0, 1)[i % 2])


@pytest.mark.parametrize("variant", ("stale", "lost_transfer", "torn_transfer", "torn_pair", "split_amount"))
def test_mutated_histories(gpu_ctx, variant):
    for p_info in (0.0, 0.02):
        spec = synth.SynthSpec("bank", 10**4, 32, 1, n_accounts=8, final_reads=True, tau_think_ns=0.0, p_info=p_info,
                               stale_read=variant == "stale")
        h = synth.generate_ledger_lookups(spec, **({} if variant == "stale" else {variant: True}))
        g = agree(gpu_ctx, h)   # a VALID is a proof the verifier accepts (split_amount at p_info 0.02 is one)
        if variant != "split_amount" or p_info == 0.0:
            assert g["valid"] != H.VALID


def test_multi_shard(gpu_ctx):
    """Shards K15 proves, shards only the class pass proves, and shards that fail or stop, in one call."""
    parts = [flat(script(CROWDED)[0]), flat(script(crowded(stale=True))[0]), flat(script(LIFTED)[0]),
             flat(script(CYCLING)[0]), flat(script(crowded(n_t=150, seen=140, n_r=140))[0])]
    parts += [synth.generate_ledger_lookups(synth.SynthSpec("bank", 10**4, 32, s, n_accounts=8, final_reads=True,
                                                            tau_think_ns=0.0, p_info=0.02)) for s in (1, 2)]
    parts += [h for _, h, kw, _ in hand_histories() if not kw]
    h = H.concat_keys(parts)
    for mr, ml, rounds in ((0, 0, 0), (1, 1, 0), (0, 0, 1)):
        g = agree(gpu_ctx, h, max_repairs=mr, max_lifts=ml, max_rounds=rounds)
        assert len(g["shards"]) == len(parts)
    s = agree(gpu_ctx, h)["shards"]
    assert s[0]["valid"] == s[4]["valid"] == H.VALID and s[0]["n_handed"] == 200 and s[4]["n_handed"] == 140
    agree_lw(gpu_ctx, h)


def test_errors_leave_the_context_usable(gpu_ctx):
    good = flat(script(CROWDED)[0])
    with pytest.raises(NativeError, match="negative amount"):
        gpu_ctx.check_class_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]), witness=True)
    assert agree(gpu_ctx, good)["valid"] == H.VALID
    with pytest.raises(NativeError, match="reserved"):
        gpu_ctx.check_class_witness(good, flags=1)
    ch = H.as_c_history(good)
    res = abi.CCwResult()
    assert native.lib().jtb_check_class_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 0, 0, 0, None, None,
                                                C.addressof(res)) < 0
    assert "null" in gpu_ctx._err()
    assert agree(gpu_ctx, good)["valid"] == H.VALID
    assert gpu_ctx.check_class_witness(good)["shards"] == agree(gpu_ctx, good)["shards"]   # without commit_read


def test_checker_result_map(gpu_ctx):
    from jepsen_tigerbeetle_b200 import checker
    r = checker.independent_checker(checker.class_witness_checker(ctx=gpu_ctx)).check({}, H.concat_keys(
        [flat(script(CROWDED)[0]), flat(script(LIFTED)[0])]))
    assert r["valid?"] is True


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkClassWitness through the JNI shim and a fake JNIEnv returns what ctypes returns."""
    fj = cw_fakejvm()
    handle = fj.create()
    try:
        parts = [flat(script(CROWDED)[0]), flat(script(crowded(stale=True))[0]), flat(script(CONFLICT)[0])]
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_class_witness(handle, fj.jhistory(h), 0, 0, 0, 0), np.int64)
        g = gpu_ctx.check_class_witness(h)
        assert v[:15].tolist() == [g[k] for k in abi.CW_RESULT_FIELDS[:15]]
        assert v[17] == h.n_shards
        for s, q in enumerate(g["shards"]):
            assert v[18 + 18 * s: 36 + 18 * s].tolist() == [q[f] for f in abi.CW_SHARD_FIELDS]
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_class_witness(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])),
                                                       0, 0, 0, 0), np.int64)
    finally:
        fj.lib().fj_destroy(handle)
