"""The counter-bounds check on the GPU (K8) against the CPU oracles, field by field: verdict, counts, witness read, key,
kind, value, bound and culprit transfer."""
import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from test_counter_bounds_cpu import UNSEEN, random_tiny
from test_monotonic_cpu import flat, inv_r, random_history, rd, tr

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_violations", "shards")


def agree(ctx, h, algo=M.CB_SWEEP):
    g = ctx.check_counter_bounds(h)
    o = M.check_counter_bounds(h, algo)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    return g


def test_random_histories(gpu_ctx):
    rng = np.random.default_rng(31)
    verdicts = set()
    for _ in range(300):
        verdicts.add(agree(gpu_ctx, flat(random_tiny(rng)[0]), M.CB_LITERAL)["valid"])
    for _ in range(100):
        verdicts.add(agree(gpu_ctx, random_history(rng, int(rng.integers(2, 30))), M.CB_LITERAL)["valid"])
    assert verdicts == {H.VALID, H.INVALID}


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("variant", ["valid", "stale", "fractured", "lost", "duplicated"])
def test_c3_size_ledger_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, stale_read=variant == "stale", final_reads=True)
    h = synth.generate_ledger_counters(spec, fractured=variant == "fractured", lost_transfer=variant == "lost",
                                       duplicated_transfer=variant == "duplicated")
    g = agree(gpu_ctx, h)
    assert g["n_reads"] > 4000
    if variant == "valid":
        assert g["valid"] == H.VALID
    if variant in ("lost", "duplicated"):
        assert g["valid"] == H.INVALID
        assert g["shards"][0]["kind"] == (abi.CB_BELOW if variant == "lost" else abi.CB_ABOVE)


def test_c3_with_crashed_transfers(gpu_ctx):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True))
    assert np.count_nonzero(h.type == H.T_INFO) > 100
    assert agree(gpu_ctx, h)["valid"] == H.VALID


@pytest.mark.parametrize("lost", [False, True])
def test_64_accounts(gpu_ctx, lost):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, p_info=0.02,
                                                       final_reads=True), lost_transfer=lost)
    g = agree(gpu_ctx, h, M.CB_LITERAL)
    assert g["shards"][0]["n_keys"] == 128
    assert g["valid"] == (H.INVALID if lost else H.VALID)


def test_multi_shard_with_one_poisoned_shard(gpu_ctx):
    parts = [synth.generate_ledger_counters(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, final_reads=True))
             for s in range(1, 9)]
    parts[5] = synth.generate_ledger_counters(synth.SynthSpec("bank", 1500, 8, 6, tau_think_ns=5e6, final_reads=True),
                                              lost_transfer=True)
    g = agree(gpu_ctx, H.concat_keys(parts), M.CB_LITERAL)
    assert [s["valid"] for s in g["shards"]] == [H.VALID] * 5 + [H.INVALID] + [H.VALID] * 2
    assert g["n_failures"] == 1


@pytest.mark.parametrize("lost", [False, True])
def test_million_op_single_shard(gpu_ctx, lost):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 1_000_000, 32, 1, final_reads=True),
                                       lost_transfer=lost)
    assert h.n_shards == 1 and h.n_events == 2_000_002
    g = agree(gpu_ctx, h)
    assert g["valid"] == (H.INVALID if lost else H.VALID) and g["n_reads"] > 400_000


def test_lost_transfer_passes_k7_and_fails_here(gpu_ctx):
    """A lost transfer keeps every read consistent with every other read: K7 passes it, this check does not."""
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 3000, 16, 2, tau_think_ns=5e6, final_reads=True),
                                       lost_transfer=True)
    assert gpu_ctx.check_monotonic_keys(h)["valid"] == H.VALID
    assert agree(gpu_ctx, h)["valid"] == H.INVALID


def test_errors_leave_the_context_usable(gpu_ctx):
    with pytest.raises(NativeError, match="negative amount"):
        gpu_ctx.check_counter_bounds(flat([tr(0, "invoke", 1, 2, -1), tr(0, "ok", 1, 2, -1)]))
    with pytest.raises(NativeError, match="outside"):
        gpu_ctx.check_counter_bounds(flat([tr(0, "invoke", -1, 2, 1)]))
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload_len[1] = 5
    with pytest.raises(NativeError, match="multiple of 3"):
        gpu_ctx.check_counter_bounds(h)
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload[3] = h.payload[0]
    with pytest.raises(NativeError, match="twice"):
        gpu_ctx.check_counter_bounds(h)
    import ctypes as C
    from jepsen_tigerbeetle_b200 import native
    h = flat([inv_r(0, [1]), rd(0, {1: (0, 0)})])
    ch = H.as_c_history(h)
    shards, res = (abi.CCbShard * 1)(), abi.CCbResult()
    assert native.lib().jtb_check_counter_bounds(gpu_ctx._h, C.addressof(ch), 1, C.addressof(shards),
                                                 C.addressof(res)) < 0
    assert "reserved" in gpu_ctx._err()
    assert agree(gpu_ctx, flat([tr(0, "invoke", 1, 2, 1), tr(0, "ok", 1, 2, 1), inv_r(1, [1, 2]),
                                rd(1, {1: (1, 0), 2: (0, 1)})]))["valid"] == H.VALID


def test_checker_result_map(gpu_ctx):
    ops = [tr(0, "invoke", 1, 2, 3), tr(0, "ok", 1, 2, 3), tr(0, "invoke", 2, 3, 1), tr(0, "ok", 2, 3, 1),
           inv_r(0, [1, 2, 3]), rd(0, {1: (3, 0), 2: (0, 3), 3: (0, 0)})]
    ops = [dict(o, index=i) for i, o in enumerate(ops)]
    r = checker.counter_bounds_checker(ctx=gpu_ctx).check({}, ops)
    assert r["valid?"] is False and (r["read-count"], r["transfer-count"], r["error-count"]) == (1, 2, 2)
    assert r["op"] == {"index": 5}
    assert r["error"] == {"type": "below-completed-transfers", "key": [2, "debits-posted"], "value": 0, "bound": 1,
                          "transfer": {"index": 3}}
    comp = checker.ledger_checker(ctx=gpu_ctx, linear=False, counter_bounds=True).check({"accounts": [1, 2, 3]}, ops)
    assert comp["counter-bounds"]["valid?"] is False and comp["valid?"] is False
    assert "counter-bounds" not in checker.ledger_checker(ctx=gpu_ctx, linear=False).check({"accounts": [1, 2, 3]},
                                                                                            ops)
    ok = [dict(o, index=i) for i, o in enumerate([tr(0, "invoke", 1, 2, 1), inv_r(1, [1, 2]), rd(1, UNSEEN)])]
    r = checker.counter_bounds_checker(ctx=gpu_ctx).check({}, ok)
    assert r["valid?"] is True and "error" not in r and "op" not in r


def test_independent_keys(gpu_ctx):
    parts = [synth.generate_ledger_counters(synth.SynthSpec("bank", 600, 8, s, tau_think_ns=5e6, final_reads=True),
                                            duplicated_transfer=s == 2) for s in (1, 2, 3)]
    h = H.concat_keys(parts)
    r = checker.independent_checker(checker.counter_bounds_checker(ctx=gpu_ctx)).check({}, h)
    assert r["valid?"] is False and r["failures"] == [int(h.key_ids[1])]


def test_jni_shim_equals_ctypes(gpu_ctx, monkeypatch):
    """jtb.Native.checkCounterBounds through the JNI shim and a fake JNIEnv returns what the ctypes binding returns."""
    import ctypes as C
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    monkeypatch.setattr(fakejvm, "_SO", os.path.join(here, "native", "libjtb_fakejvm_cb.so"))
    monkeypatch.setattr(fakejvm, "_SRCS", [os.path.join(here, "native", "fake_jvm_cb.c")] + fakejvm._SRCS[1:])
    monkeypatch.setattr(fakejvm, "_DEPS", fakejvm._DEPS + [os.path.join(here, "native", "fake_jvm_cb.c"),
                                                           os.path.join(here, "native", "fake_jvm.c")])
    monkeypatch.setattr(fakejvm, "_lib", None)
    L = fakejvm.lib()
    L.fj_check_counter_bounds.restype = C.c_void_p
    L.fj_check_counter_bounds.argtypes = [C.c_longlong, C.c_void_p]
    handle = fakejvm.create()
    try:
        parts = [synth.generate_ledger_counters(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, final_reads=True),
                                                lost_transfer=s == 2, duplicated_transfer=s == 3) for s in (1, 2, 3)]
        h = H.concat_keys(parts)
        v = fakejvm._result(L.fj_check_counter_bounds(handle, fakejvm.jhistory(h)), np.int64)
        g = gpu_ctx.check_counter_bounds(h)
        assert v[:5].tolist() == [g["valid"], g["n_failures"], g["n_reads"], g["n_transfers"], g["n_violations"]]
        assert v[7] == h.n_shards
        for s, q in enumerate(g["shards"]):
            assert v[8 + 12 * s: 20 + 12 * s].tolist() == [q[f] for f in abi.CB_SHARD_FIELDS]
        bad = flat([tr(0, "invoke", 1, 2, -5)])
        with pytest.raises(fakejvm.JavaException, match="negative amount"):
            fakejvm._result(L.fj_check_counter_bounds(handle, fakejvm.jhistory(bad)), np.int64)
    finally:
        L.fj_destroy(handle)
