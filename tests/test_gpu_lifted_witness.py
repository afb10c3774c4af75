"""The lifted serial witness on the GPU (K15) against LW_SEARCH, field by field and commit_read entry for entry, with
every VALID proof re-checked by the independent verifier: the panel of valid bank histories, the random families, the
hand cases, a multi-shard history that mixes shards K14 proves with shards only a lift step proves, the budgets, the
error paths and the JNI shim; and K14's device results on the same inputs, which the shared repair loop must leave as
RW_SEARCH computes them."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from serial_witness import verify
from test_lifted_witness_cpu import CYCLING, LIFTED, lw_fakejvm
from test_repaired_witness_cpu import panel
from test_serial_witness_cpu import CONFLICT, hand_histories
from test_transfer_lookups_cpu import flat, random_tiny, tr
from test_transfer_placement_cpu import regrouping, script

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes",
          "rounds", "repairs", "n_bans", "lifts", "n_lifted", "shards")
RW_FIELDS = FIELDS[:11] + ("shards",)


def agree(ctx, h, max_nodes=0, max_rounds=0, max_repairs=0, max_lifts=0):
    g = ctx.check_lifted_witness(h, max_nodes, max_rounds, max_repairs, max_lifts, witness=True)
    o = M.check_lifted_witness(h, max_nodes=max_nodes, max_rounds=max_rounds, max_repairs=max_repairs,
                               max_lifts=max_lifts)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    assert np.array_equal(g["commit_read"], o["commit_read"])
    verify(h, g)
    return g


def agree_rw(ctx, h, **kw):
    g = ctx.check_repaired_witness(h, witness=True, **kw)
    o = M.check_repaired_witness(h, **kw)
    assert {k: g[k] for k in RW_FIELDS} == {k: o[k] for k in RW_FIELDS}
    assert np.array_equal(g["commit_read"], o["commit_read"])
    return g


def lifted_panel():
    """The 10^5-op, 8-account panel histories whose K14 repairs stop and that lift steps prove."""
    return [h for (ops, n, p, seed), h in panel(10**5).items() if n == 8 and (p, seed) != (0.0, 2)]


@pytest.mark.parametrize("ops", [10**4, 10**5])
def test_panel(gpu_ctx, ops):
    for key, h in panel(ops).items():
        g = agree(gpu_ctx, h)
        agree_rw(gpu_ctx, h)
        s = g["shards"][0]
        print(key, abi.CAUSE_NAME.get(s["cause"], "VALID"), "repairs", s["repairs"], "lifts", s["lifts"], "lifted",
              s["n_lifted"], "bans", s["n_bans"])


def test_budgets(gpu_ctx):
    h = lifted_panel()[0]
    assert agree(gpu_ctx, h)["valid"] == H.VALID
    for ml in (1, 2):
        agree(gpu_ctx, h, max_lifts=ml)
    for mr in (1, 7):
        agree(gpu_ctx, h, max_repairs=mr)
    agree(gpu_ctx, h, max_rounds=1)
    agree(gpu_ctx, h, max_nodes=3)


def test_hand_cases(gpu_ctx):
    for steps in (LIFTED, CYCLING):
        h = flat(script(steps)[0])
        for ml in (0, 1):
            agree(gpu_ctx, h, max_lifts=ml)
        agree_rw(gpu_ctx, h)
    assert agree(gpu_ctx, flat(script(LIFTED)[0]))["valid"] == H.VALID
    for name, h, kw, cause in hand_histories():
        agree(gpu_ctx, h, **kw)


def test_random_histories(gpu_ctx):
    rng = np.random.default_rng(113)
    for i in range(200):
        agree(gpu_ctx, flat(random_tiny(rng)[0]), max_nodes=(0, 1, 3)[i % 3], max_rounds=(0, 1, 2)[i % 3 - 1])
        agree(gpu_ctx, flat(regrouping(rng)[0]), max_repairs=(0, 1)[i % 2], max_lifts=(0, 1)[i % 2])


@pytest.mark.parametrize("variant", ("stale", "lost_transfer", "torn_transfer", "torn_pair", "split_amount"))
def test_mutated_histories(gpu_ctx, variant):
    spec = synth.SynthSpec("bank", 10**4, 32, 1, n_accounts=8, final_reads=True, tau_think_ns=0.0,
                           stale_read=variant == "stale")
    h = synth.generate_ledger_lookups(spec, **({} if variant == "stale" else {variant: True}))
    assert agree(gpu_ctx, h)["valid"] != H.VALID


def test_multi_shard(gpu_ctx):
    """Shards K14 proves, shards only a lift step proves, and shards that fail or stop, in one call."""
    muts = {2: "torn_transfer", 5: "split_amount"}
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05,
                                                           final_reads=True), **({muts[s]: True} if s in muts else {}))
             for s in range(1, 7)]
    parts += [synth.generate_ledger_lookups(synth.SynthSpec("bank", 10**4, 32, 1, n_accounts=8, final_reads=True,
                                                            tau_think_ns=0.0))]
    parts += lifted_panel()
    parts += [flat(script(LIFTED)[0]), flat(script(CYCLING)[0])]
    parts += [h for _, h, kw, _ in hand_histories() if not kw]
    h = H.concat_keys(parts)
    for mr, ml in ((0, 0), (1, 0), (0, 1), (6, 2)):
        g = agree(gpu_ctx, h, max_repairs=mr, max_lifts=ml)
        assert len(g["shards"]) == len(parts)
    assert sum(s["lifts"] > 0 and s["valid"] == H.VALID for s in agree(gpu_ctx, h)["shards"]) >= 3
    agree_rw(gpu_ctx, h)


def test_errors_leave_the_context_usable(gpu_ctx):
    good = flat(script(LIFTED)[0])
    with pytest.raises(NativeError, match="negative amount"):
        gpu_ctx.check_lifted_witness(flat([tr(0, "invoke", 1, 2, -1, 1)]), witness=True)
    assert agree(gpu_ctx, good)["valid"] == H.VALID
    with pytest.raises(NativeError, match="reserved"):
        gpu_ctx.check_lifted_witness(good, flags=1)
    ch = H.as_c_history(good)
    res = abi.CLwResult()
    assert native.lib().jtb_check_lifted_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 0, 0, 0, None, None,
                                                 C.addressof(res)) < 0
    assert "null" in gpu_ctx._err()
    assert agree(gpu_ctx, good)["valid"] == H.VALID
    assert gpu_ctx.check_lifted_witness(good)["shards"] == agree(gpu_ctx, good)["shards"]   # without commit_read


def test_checker_result_map(gpu_ctx):
    from jepsen_tigerbeetle_b200 import checker
    r = checker.independent_checker(checker.lifted_witness_checker(ctx=gpu_ctx)).check({}, H.concat_keys(
        lifted_panel()[:2]))
    assert r["valid?"] is True


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkLiftedWitness through the JNI shim and a fake JNIEnv returns what ctypes returns."""
    fj = lw_fakejvm()
    handle = fj.create()
    try:
        parts = [flat(script(LIFTED)[0]), flat(script(CYCLING)[0]), flat(script(CONFLICT)[0])]
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_lifted_witness(handle, fj.jhistory(h), 0, 0, 0, 0), np.int64)
        g = gpu_ctx.check_lifted_witness(h)
        assert v[:13].tolist() == [g[k] for k in abi.LW_RESULT_FIELDS[:13]]
        assert v[15] == h.n_shards
        for s, q in enumerate(g["shards"]):
            assert v[16 + 15 * s: 31 + 15 * s].tolist() == [q[f] for f in abi.LW_SHARD_FIELDS]
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_lifted_witness(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])),
                                                        0, 0, 0, 0), np.int64)
    finally:
        fj.lib().fj_destroy(handle)
