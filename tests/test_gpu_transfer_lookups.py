"""The transfer-lookup check on the GPU (K9) against the CPU oracles, field by field: verdict, counts by kind, witness
op, kind, transfer id, key, value, bound and related op; K7 and K8 on the lookups form; every error path."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from test_monotonic_cpu import inv_r, rd
from test_transfer_lookups_cpu import R1, T1, _tl_fakejvm, flat, inv_l, lk, ops_idx, random_tiny, tr

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_lookups", "n_records", "n_transfers", "n_reads", "n_violations", "shards")
MUTATIONS = ("lost_transfer", "phantom_record", "mismatched_record", "vanished_record", "inflated_read")


def agree(ctx, h, algo=M.TL_SWEEP):
    g = ctx.check_transfer_lookups(h)
    o = M.check_transfer_lookups(h, algo)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    return g


def test_random_tiny_histories(gpu_ctx):
    rng = np.random.default_rng(37)
    kinds = set()
    for _ in range(400):
        g = agree(gpu_ctx, flat(random_tiny(rng)[0]), M.TL_LITERAL)
        kinds.add(g["shards"][0]["kind"])
    assert len(kinds) >= 6, kinds


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("variant", ("valid",) + MUTATIONS)
def test_c3_size_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, final_reads=True, p_info=0.02 if variant == "vanished_record" else 0)
    h = synth.generate_ledger_lookups(spec, **({} if variant == "valid" else {variant: True}))
    g = agree(gpu_ctx, h)
    assert g["n_lookups"] == 32 and g["valid"] == (H.VALID if variant == "valid" else H.INVALID)


def test_crashed_transfers(gpu_ctx):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True))
    assert np.count_nonzero(h.type == H.T_INFO) > 100
    assert agree(gpu_ctx, h)["valid"] == H.VALID


def test_mid_history_lookups(gpu_ctx):
    for seed in (1, 2):
        spec = synth.SynthSpec("bank", 600, 8, seed, p_info=0.05, final_reads=True)
        for kw in ({}, {"lost_transfer": True}, {"inflated_read": True}):
            agree(gpu_ctx, synth.generate_ledger_lookups(spec, p_lookup=0.05, **kw), M.TL_LITERAL)


@pytest.mark.parametrize("lost", [False, True])
def test_64_accounts(gpu_ctx, lost):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, p_info=0.02,
                                                      final_reads=True), lost_transfer=lost)
    g = agree(gpu_ctx, h, M.TL_LITERAL)
    assert g["valid"] == (H.INVALID if lost else H.VALID)


def test_multi_shard_with_poisoned_shards(gpu_ctx):
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05,
                                                           final_reads=True),
                                           **({MUTATIONS[s % 5]: True} if s in (2, 5, 6) else {}))
             for s in range(1, 9)]
    g = agree(gpu_ctx, H.concat_keys(parts), M.TL_LITERAL)
    assert [s["valid"] for s in g["shards"]] == [H.INVALID if s in (2, 5, 6) else H.VALID for s in range(1, 9)]


@pytest.mark.parametrize("lost", [False, True])
def test_million_op_history(gpu_ctx, lost):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 1_000_000, 32, 1, final_reads=True),
                                      lost_transfer=lost)
    g = agree(gpu_ctx, h)
    assert g["n_lookups"] == 32 and g["n_records"] > 32 * 400_000
    assert g["valid"] == (H.INVALID if lost else H.VALID)


@pytest.mark.parametrize("kw", [{}, {"lost_transfer": True}, {"inflated_read": True}])
def test_k7_and_k8_ignore_the_lookups(gpu_ctx, kw):
    spec = synth.SynthSpec("bank", 3000, 16, 2, tau_think_ns=5e6, p_info=0.02, final_reads=True)
    h = synth.generate_ledger_lookups(spec, **kw)
    c = synth.generate_ledger_counters(spec, lost_transfer=kw.get("lost_transfer", False))
    if kw.get("inflated_read"):   # the same mutation on the counter form
        e = np.nonzero((c.flags & H.FLAG_FINAL).astype(bool) & (c.type == H.T_OK))[0][0]
        c.payload[c.payload_off[e] + 1] += 1
    strip = lambda r: {k: v for k, v in r.items() if not k.startswith("seconds")}   # noqa: E731
    assert strip(gpu_ctx.check_monotonic_keys(h)) == strip(gpu_ctx.check_monotonic_keys(c))
    assert strip(gpu_ctx.check_counter_bounds(h)) == strip(gpu_ctx.check_counter_bounds(c))


def test_errors_leave_the_context_usable(gpu_ctx):
    def raises(ops, match, mutate=None):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(NativeError, match=match):
            gpu_ctx.check_transfer_lookups(h)
        assert agree(gpu_ctx, flat(T1 + [inv_l(1), lk(1, [R1])]))["valid"] == H.VALID

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", -1, 2, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, 0))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises(T1 + [inv_l(1), lk(1, [R1])], "multiple of 5", lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "multiple of 3", lambda h: h.payload_len.__setitem__(1, 5))
    h = flat(T1)
    ch = H.as_c_history(h)
    shards, res = (abi.CTlShard * 1)(), abi.CTlResult()
    assert native.lib().jtb_check_transfer_lookups(gpu_ctx._h, C.addressof(ch), 1, C.addressof(shards),
                                                   C.addressof(res)) < 0
    assert "reserved" in gpu_ctx._err()
    assert agree(gpu_ctx, flat(T1 + [inv_l(1), lk(1, [])]))["valid"] == H.INVALID


def test_checker_result_map(gpu_ctx):
    ops = ops_idx(T1 + [inv_l(1), lk(1, [])])
    r = checker.transfer_lookup_checker(ctx=gpu_ctx).check({}, ops)
    assert r["valid?"] is False and r["errors"] == {"lost": 1} and r["op"] == {"index": 3}
    assert r["error"] == {"type": "lost", "transfer-id": 1, "related": {"index": 1}}
    comp = checker.ledger_checker(ctx=gpu_ctx, linear=False, transfer_lookups=True).check({"accounts": [1, 2]}, ops)
    assert comp["transfer-lookups"]["valid?"] is False and comp["valid?"] is False
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 600, 8, s, tau_think_ns=5e6, final_reads=True),
                                           phantom_record=s == 2) for s in (1, 2, 3)]
    h = H.concat_keys(parts)
    r = checker.independent_checker(checker.transfer_lookup_checker(ctx=gpu_ctx)).check({}, h)
    assert r["valid?"] is False and r["failures"] == [int(h.key_ids[1])]


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkTransferLookups through the JNI shim and a fake JNIEnv returns what the ctypes binding returns."""
    fj = _tl_fakejvm()
    handle = fj.create()
    try:
        parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, final_reads=True),
                                               lost_transfer=s == 2, mismatched_record=s == 3) for s in (1, 2, 3)]
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_transfer_lookups(handle, fj.jhistory(h)), np.int64)
        g = gpu_ctx.check_transfer_lookups(h)
        assert v[:7].tolist() == [g[k] for k in ("valid", "n_failures", "n_lookups", "n_records", "n_transfers",
                                                 "n_reads", "n_violations")]
        assert v[9] == h.n_shards
        for s, q in enumerate(g["shards"]):
            want = [q["valid"], q["n_lookups"], q["n_records"], q["n_transfers"], q["n_reads"]] + q["count_by_kind"] + [
                q[f] for f in ("witness_index", "kind", "transfer_id", "key", "related_index", "value", "bound")]
            assert v[10 + 21 * s: 31 + 21 * s].tolist() == want
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_transfer_lookups(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)]))),
                       np.int64)
    finally:
        fj.lib().fj_destroy(handle)
