"""The monotonic-key check on the GPU (K7) against the MONO_GRAPH oracle, field by field: verdict, cause, counts,
witness, partner and both edge explanations."""
import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from test_monotonic_cpu import flat, inv_r, random_history, rd

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "shards")


def same(g, o):
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}


def agree(ctx, h, realtime=True):
    g = ctx.check_monotonic_keys(h, realtime=realtime)
    o = M.check_monotonic_keys(h, M.MONO_GRAPH, realtime=realtime)
    same(g, o)
    return g


@pytest.mark.parametrize("realtime", [True, False])
def test_random_histories(gpu_ctx, realtime):
    rng = np.random.default_rng(11 if realtime else 12)
    verdicts = set()
    for _ in range(300):
        verdicts.add(agree(gpu_ctx, random_history(rng, int(rng.integers(2, 30))), realtime)["valid"])
    assert verdicts == {H.VALID, H.INVALID}


def test_random_histories_as_one_keyed_history(gpu_ctx):
    rng = np.random.default_rng(13)
    parts = [random_history(rng, int(rng.integers(2, 30))) for _ in range(64)]
    g = agree(gpu_ctx, H.concat_keys(parts))
    assert 0 < g["n_failures"] < 64


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("variant", ["valid", "stale", "fractured"])
def test_c3_size_ledger_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, stale_read=variant == "stale")
    h = synth.generate_ledger_counters(spec, fractured=variant == "fractured")
    for rt in (True, False):
        g = agree(gpu_ctx, h, rt)
        if variant == "valid":
            assert g["valid"] == H.VALID   # linearizable by construction
    assert g["n_reads"] > 4000


def test_c3_with_crashed_transfers(gpu_ctx):
    """C3 with p_info 0.02: the linearizability search leaves it :unknown; this check decides it."""
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02))
    assert np.count_nonzero(h.type == H.T_INFO) > 100
    assert agree(gpu_ctx, h)["valid"] == H.VALID
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, stale_read=True))
    agree(gpu_ctx, h)


@pytest.mark.parametrize("stale", [False, True])
def test_64_accounts(gpu_ctx, stale):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, p_info=0.02,
                                                       stale_read=stale))
    g = agree(gpu_ctx, h)
    assert g["shards"][0]["n_keys"] == 128


def test_multi_shard_with_one_poisoned_shard(gpu_ctx):
    parts = [synth.generate_ledger_counters(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6)) for s in range(1, 9)]
    parts[5] = synth.generate_ledger_counters(synth.SynthSpec("bank", 1500, 8, 6, tau_think_ns=5e6), fractured=True)
    h = H.concat_keys(parts)
    g = agree(gpu_ctx, h)
    assert [s["valid"] for s in g["shards"]] == [H.VALID] * 5 + [H.INVALID] + [H.VALID] * 2
    assert g["n_failures"] == 1


def test_million_op_single_shard(gpu_ctx):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 1_000_000, 32, 1, p_info=0.02))
    assert h.n_shards == 1 and h.n_events == 2_000_000
    g = agree(gpu_ctx, h)
    assert g["valid"] == H.VALID and g["n_reads"] > 400_000


def test_million_op_stale_read(gpu_ctx):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 1_000_000, 32, 1, stale_read=True, stale_frac=0.5))
    assert agree(gpu_ctx, h)["valid"] == H.INVALID


def test_partial_reads_are_unknown(gpu_ctx):
    ops = [inv_r(0, [1, 2]), inv_r(1, [2, 3]), inv_r(2, [3, 1]),
           rd(0, {1: (1, 1), 2: (0, 0)}), rd(1, {2: (1, 1), 3: (0, 0)}), rd(2, {3: (1, 1), 1: (0, 0)})]
    g = agree(gpu_ctx, flat(ops))
    assert (g["valid"], g["shards"][0]["cause"]) == (H.UNKNOWN, abi.CAUSE_PARTIAL_READ)
    # one account with nil amounts makes a read partial
    g = agree(gpu_ctx, flat([inv_r(0, [1, 2]), rd(0, {1: (1, 0), 2: None}), inv_r(0, [1, 2]), rd(0, {1: (1, 0), 2: (0, 0)})]))
    assert g["shards"][0]["cause"] == abi.CAUSE_PARTIAL_READ


def test_no_realtime_flag(gpu_ctx):
    ops = [inv_r(0, [1]), rd(0, {1: (2, 0)}), inv_r(1, [1]), rd(1, {1: (1, 0)})]
    assert agree(gpu_ctx, flat(ops), True)["valid"] == H.INVALID
    assert agree(gpu_ctx, flat(ops), False)["valid"] == H.VALID


def test_malformed_payloads_are_errors(gpu_ctx):
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload_len[1] = 5
    with pytest.raises(NativeError, match="multiple of 3"):
        gpu_ctx.check_monotonic_keys(h)
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload[3] = h.payload[0]
    with pytest.raises(NativeError, match="twice"):
        gpu_ctx.check_monotonic_keys(h)
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload_off[1] = 1 << 40
    with pytest.raises(NativeError, match="out of range"):
        gpu_ctx.check_monotonic_keys(h)
    # the context is still usable
    assert gpu_ctx.check_monotonic_keys(flat([inv_r(0, [1]), rd(0, {1: (1, 0)})]))["valid"] == H.VALID


def test_checker_result_map(gpu_ctx):
    ops = [inv_r(0, [1, 2]), inv_r(1, [1, 2]), rd(0, {1: (1, 0), 2: (0, 0)}), rd(1, {1: (0, 0), 2: (1, 0)})]
    ops = [dict(o, index=i) for i, o in enumerate(ops)]
    r = checker.monotonic_key_checker(ctx=gpu_ctx).check({}, ops)
    assert r["valid?"] is False and r["read-count"] == 2 and r["key-count"] == 4
    assert r["op"] == {"index": 3} and r["cycle"] == [{"index": 2}, {"index": 3}, {"index": 2}]
    assert r["steps"] == [{"type": "monotonic", "key": [2, "debits-posted"], "value": 0, "value'": 1},
                          {"type": "monotonic", "key": [1, "debits-posted"], "value": 0, "value'": 1}]
    comp = checker.ledger_checker(ctx=gpu_ctx, linear=False, monotonic=True).check({"accounts": [1, 2]}, ops)
    assert comp["monotonic"]["valid?"] is False
    assert "monotonic" not in checker.ledger_checker(ctx=gpu_ctx, linear=False).check({"accounts": [1, 2]}, ops)


def test_jni_shim_equals_ctypes(gpu_ctx, monkeypatch):
    """jtb.Native.checkMonotonicKeys through the JNI shim and a fake JNIEnv returns what the ctypes binding returns."""
    import ctypes as C
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    monkeypatch.setattr(fakejvm, "_SO", os.path.join(here, "native", "libjtb_fakejvm_mono.so"))
    monkeypatch.setattr(fakejvm, "_SRCS", [os.path.join(here, "native", "fake_jvm_mono.c")] + fakejvm._SRCS[1:])
    monkeypatch.setattr(fakejvm, "_DEPS", fakejvm._DEPS + [os.path.join(here, "native", "fake_jvm_mono.c"),
                                                           os.path.join(here, "native", "fake_jvm.c")])
    monkeypatch.setattr(fakejvm, "_lib", None)
    L = fakejvm.lib()
    L.fj_check_monotonic_keys.restype = C.c_void_p
    L.fj_check_monotonic_keys.argtypes = [C.c_longlong, C.c_void_p, C.c_int]
    handle = fakejvm.create()
    try:
        parts = [synth.generate_ledger_counters(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6), fractured=s == 2)
                 for s in (1, 2, 3)]
        h = H.concat_keys(parts)
        for rt in (True, False):
            v = fakejvm._result(L.fj_check_monotonic_keys(handle, fakejvm.jhistory(h), int(rt)), np.int64)
            g = gpu_ctx.check_monotonic_keys(h, realtime=rt)
            assert v[:3].tolist() == [g["valid"], g["n_failures"], g["n_reads"]] and v[5] == h.n_shards
            for s, q in enumerate(g["shards"]):
                rec = v[6 + 14 * s: 20 + 14 * s].tolist()
                assert rec[:6] == [q[f] for f in abi.MONO_SHARD_FIELDS]
                assert [tuple(rec[6:10]), tuple(rec[10:14])] == q["edges"]
        bad = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
        bad.payload_len[1] = 4
        with pytest.raises(fakejvm.JavaException, match="multiple of 3"):
            fakejvm._result(L.fj_check_monotonic_keys(handle, fakejvm.jhistory(bad), 1), np.int64)
    finally:
        L.fj_destroy(handle)
