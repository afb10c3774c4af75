"""The lookup witness on the GPU (K17) against LK_SEARCH, field by field, commit_read and lookup_read entry for entry,
with every VALID proof re-checked by the independent verifier: the hand cases, the panel of valid bank histories,
generated histories with mid-run lookups, the random families, the mutations that must never be VALID, lookup-free
histories (equal to the class witness on the device), the ABI sizes, the NULL outputs and the JNI shim."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, native, synth
from jepsen_tigerbeetle_b200 import history as H
from lookup_witness import verify
from test_class_witness_cpu import CROWDED
from test_lookup_witness_cpu import CROSSING, EARLY, lk_fakejvm, regrouping_lookups
from test_repaired_witness_cpu import panel
from test_transfer_lookups_cpu import flat, random_tiny, tr
from test_transfer_placement_cpu import script

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes",
          "rounds", "repairs", "n_bans", "lifts", "n_lifted", "class_rounds", "n_handed", "n_lookups_placed", "shards")


def agree(ctx, h, **kw):
    g = ctx.check_lookup_witness(h, witness=True, **kw)
    o = M.check_lookup_witness(h, **kw)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    assert np.array_equal(g["commit_read"], o["commit_read"])
    assert np.array_equal(g["lookup_read"], o["lookup_read"])
    verify(h, g)
    return g


def test_hand_cases(gpu_ctx):
    assert agree(gpu_ctx, flat(script(CROWDED)[0]))["valid"] == H.VALID
    steps = CROWDED[:-1] + [("l", [f"x{k}" for k in range(210)])]
    g = agree(gpu_ctx, flat(script(steps)[0]))
    assert g["valid"] == H.VALID and (g["commit_read"][200:210] == abi.SW_AFTER).all()
    for h in (flat(script(CROSSING)[0]), flat(EARLY)):
        s = agree(gpu_ctx, h)["shards"][0]
        assert (s["valid"], s["lookup_cause"]) == (H.UNKNOWN, abi.CAUSE_LOOKUP)


@pytest.mark.parametrize("ops", [10**4, 10**5])
def test_panel(gpu_ctx, ops):
    for key, h in panel(ops).items():
        g = agree(gpu_ctx, h)
        cw = gpu_ctx.check_class_witness(h)
        if cw["valid"] == H.VALID:   # final lookups only: what K16 proves, K17 proves
            assert g["valid"] == H.VALID, key


@pytest.mark.parametrize("p_lookup", [0.0, 0.01, 0.05])
@pytest.mark.parametrize("p_info", [0.0, 0.02])
def test_generated(gpu_ctx, p_lookup, p_info):
    for seed in (1, 2, 3):
        spec = synth.SynthSpec("bank", 2000, 16, seed, n_accounts=8, final_reads=True, tau_think_ns=0.0,
                               p_info=p_info)
        agree(gpu_ctx, synth.generate_ledger_lookups(spec, p_lookup=p_lookup))


@pytest.mark.parametrize("variant", ["phantom_record", "mismatched_record", "vanished_record", "lost_transfer",
                                     "inflated_read"])
def test_mutations_are_never_valid(gpu_ctx, variant):
    for seed in (1, 2):
        for p_info in (0.02,) if variant == "vanished_record" else (0.0, 0.02):   # it drops a committed :info one
            spec = synth.SynthSpec("bank", 10**4, 32, seed, n_accounts=8, final_reads=True, tau_think_ns=0.0,
                                   p_info=p_info)
            h = synth.generate_ledger_lookups(spec, **{variant: True})
            assert agree(gpu_ctx, h)["valid"] != H.VALID


@pytest.mark.parametrize("gen", ["tiny", "regrouping"])
def test_random_histories(gpu_ctx, gen):
    rng = np.random.default_rng(131 if gen == "tiny" else 137)
    hs = [flat((random_tiny(rng) if gen == "tiny" else regrouping_lookups(rng))[0]) for _ in range(300)]
    g = agree(gpu_ctx, H.concat_keys(hs))
    assert g["n_lookups_placed"] > 0


def test_lookup_free_equals_class_witness(gpu_ctx):
    rng = np.random.default_rng(139)
    ops = []
    for _ in range(200):
        o, _ = random_tiny(rng)
        ops.append(flat([x for x in o if x["value"] and not any(m[0] == "l-t" for m in x["value"])]))
    h = H.concat_keys(ops)
    g = gpu_ctx.check_lookup_witness(h, witness=True)
    c = gpu_ctx.check_class_witness(h, witness=True)
    assert {f: g[f] for f in abi.CW_RESULT_FIELDS if not f.startswith("seconds")} == \
        {f: c[f] for f in abi.CW_RESULT_FIELDS if not f.startswith("seconds")}
    assert [{f: s[f] for f in abi.CW_SHARD_FIELDS} for s in g["shards"]] == \
        [{f: s[f] for f in abi.CW_SHARD_FIELDS} for s in c["shards"]]
    assert np.array_equal(g["commit_read"], c["commit_read"])


def test_abi_and_null_outputs(gpu_ctx):
    lib = native.lib()
    assert lib.jtb_struct_size(30) == C.sizeof(abi.CLkShard) and lib.jtb_struct_size(31) == C.sizeof(abi.CLkResult)
    h = flat(script(CROWDED)[0])
    ch = H.as_c_history(h)
    shards = (abi.CLkShard * 1)()
    res = abi.CLkResult()
    assert lib.jtb_check_lookup_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 0, 0, 0, None, None, C.addressof(shards),
                                        C.addressof(res)) == 0
    assert res.valid == H.VALID and res.n_lookups_placed == 1
    assert lib.jtb_check_lookup_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 0, 0, 0, None, None, None,
                                        C.addressof(res)) < 0
    assert lib.jtb_check_lookup_witness(gpu_ctx._h, C.addressof(ch), 0, 0, 0, 0, 1, None, None, C.addressof(shards),
                                        C.addressof(res)) < 0
    with pytest.raises(native.NativeError, match="reserved"):
        gpu_ctx.check_lookup_witness(h, flags=1)


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkLookupWitness through the JNI shim and a fake JNIEnv returns what ctypes returns."""
    fj = lk_fakejvm()
    handle = fj.create()
    try:
        h = H.concat_keys([flat(script(CROWDED)[0]), flat(script(CROSSING)[0]), flat(EARLY)])
        v = fj._result(fj.lib().fj_check_lookup_witness(handle, fj.jhistory(h), 0, 0, 0, 0), np.int64)
        g = gpu_ctx.check_lookup_witness(h)
        assert v[:16].tolist() == [g[k] for k in abi.LK_RESULT_FIELDS[:16]]
        assert v[18] == h.n_shards
        for s, q in enumerate(g["shards"]):
            assert v[19 + 21 * s: 40 + 21 * s].tolist() == [q[f] for f in abi.LK_SHARD_FIELDS]
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_lookup_witness(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])),
                                                        0, 0, 0, 0), np.int64)
    finally:
        fj.lib().fj_destroy(handle)
