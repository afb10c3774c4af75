"""The read-gap check on the GPU (K11) against RG_SEARCH, field by field: verdict, per-kind, explained and undecided
counts, node totals and the witness (ops, kind, key, Delta, transfer, other op, |eligible|); every error path; the
checker maps and the JNI shim."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from test_monotonic_cpu import inv_r, rd
from test_read_gaps_cpu import REGROUPED, _ones, _rg_fakejvm, two
from test_transfer_lookups_cpu import flat, inv_l, lk, ops_idx, random_tiny, tr

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_explained", "n_unexplained", "n_double", "n_undecided",
          "nodes", "shards")
MUTATIONS = ("torn_transfer", "torn_pair", "split_amount")
DOUBLE = [tr(0, "invoke", 1, 2, 5, 9), inv_r(1, [1, 2]), rd(1, two(5)), inv_r(1, [1, 2]), rd(1, two(10)),
          tr(0, "ok", 1, 2, 5, 9)]


def agree(ctx, h, max_nodes=0):
    g = ctx.check_read_gaps(h, max_nodes)
    o = M.check_read_gaps(h, M.RG_SEARCH, max_nodes=max_nodes)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    return g


def test_random_tiny_histories(gpu_ctx):
    rng = np.random.default_rng(59)
    kinds = set()
    for i in range(400):
        g = agree(gpu_ctx, flat(random_tiny(rng)[0]), max_nodes=(0, 1, 3)[i % 3])
        kinds.add(g["shards"][0]["kind"])
    assert kinds >= {0, abi.RG_KEY}, kinds


def test_hand_cases(gpu_ctx):
    assert agree(gpu_ctx, flat(REGROUPED))["shards"][0]["kind"] == abi.RG_KEY
    assert agree(gpu_ctx, flat(DOUBLE))["shards"][0]["kind"] == abi.RG_DOUBLE
    for n, shows in ((40, (20, 20)), (70, (35, 35)), (130, (65, 65))):   # search / free cap / gather cap
        agree(gpu_ctx, flat(_ones(n, shows)))
    for mx in (0, 1, 2, 5):
        agree(gpu_ctx, flat(_ones(40, (20, 21))), mx)
    partial = [tr(0, "invoke", 1, 2, 2, 1), inv_r(1, [1, 2]), rd(1, two(2)), inv_r(1, [2]), rd(1, {2: (0, 1)})]
    assert agree(gpu_ctx, flat(partial))["shards"][0]["cause"] == abi.CAUSE_PARTIAL_READ


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("variant", ("valid", "stale", "lost_transfer") + MUTATIONS)
def test_c3_size_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, final_reads=True, stale_read=variant == "stale")
    h = synth.generate_ledger_lookups(spec, **({variant: True} if variant in MUTATIONS + ("lost_transfer",) else {}))
    g = agree(gpu_ctx, h)
    if variant == "valid":
        assert g["n_unexplained"] == g["n_double"] == 0


def test_crashed_transfers(gpu_ctx):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True))
    assert np.count_nonzero(h.type == H.T_INFO) > 100
    g = agree(gpu_ctx, h)
    assert g["n_unexplained"] == g["n_double"] == 0 and g["n_explained"] > 0.9 * g["n_reads"]


def test_mid_history_lookups(gpu_ctx):
    spec = synth.SynthSpec("bank", 600, 8, 2, p_info=0.05, final_reads=True)
    for kw in ({}, {"lost_transfer": True}, {"torn_pair": True}):
        agree(gpu_ctx, synth.generate_ledger_lookups(spec, p_lookup=0.05, **kw))


@pytest.mark.parametrize("kw", [{}, {"torn_pair": True}])
def test_64_accounts(gpu_ctx, kw):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, p_info=0.02,
                                                      final_reads=True), **kw)
    g = agree(gpu_ctx, h)
    if not kw:
        assert g["n_unexplained"] == g["n_double"] == 0


def test_multi_shard(gpu_ctx):
    muts = {2: "torn_transfer", 5: "split_amount", 6: "torn_pair"}
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05,
                                                           final_reads=True), **({muts[s]: True} if s in muts else {}))
             for s in range(1, 9)]
    g = agree(gpu_ctx, H.concat_keys(parts))
    assert len(g["shards"]) == 8


@pytest.mark.parametrize("kw", [{}, {"torn_pair": True}])
def test_million_op_history(gpu_ctx, kw):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 1_000_000, 32, 1, final_reads=True), **kw)
    g = agree(gpu_ctx, h)
    assert g["n_reads"] > 400_000
    if not kw:
        assert g["n_unexplained"] == g["n_double"] == 0


def test_errors_leave_the_context_usable(gpu_ctx):
    ok = [tr(0, "invoke", 1, 2, 1, 1), tr(0, "ok", 1, 2, 1, 1)]

    def raises(ops, match, mutate=None):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(NativeError, match=match):
            gpu_ctx.check_read_gaps(h)
        assert agree(gpu_ctx, flat(REGROUPED))["valid"] == H.INVALID

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", -1, 2, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, 0))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises(ok + [inv_l(1), lk(1, [(1, 1, 2, 1)])], "multiple of 5", lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "multiple of 3", lambda h: h.payload_len.__setitem__(1, 5))
    h = flat(ok)
    ch = H.as_c_history(h)
    shards, res = (abi.CRgShard * 1)(), abi.CRgResult()
    assert native.lib().jtb_check_read_gaps(gpu_ctx._h, C.addressof(ch), 0, 1, C.addressof(shards),
                                            C.addressof(res)) < 0
    assert "reserved" in gpu_ctx._err()
    assert agree(gpu_ctx, flat(REGROUPED))["valid"] == H.INVALID


def test_checker_result_map(gpu_ctx):
    r = checker.read_gap_checker(ctx=gpu_ctx).check({}, ops_idx(REGROUPED))
    assert r["valid?"] is False and r["errors"] == {"key": 1} and r["op"] == {"index": 6}
    comp = checker.ledger_checker(ctx=gpu_ctx, linear=False, read_gaps=True).check({"accounts": [1, 2]},
                                                                                    ops_idx(REGROUPED))
    assert comp["read-gaps"]["valid?"] is False and comp["valid?"] is False
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 600, 8, s, tau_think_ns=5e6, final_reads=True))
             for s in (1, 2, 3)]
    h = H.concat_keys(parts)
    r = checker.independent_checker(checker.read_gap_checker(ctx=gpu_ctx)).check({}, h)
    assert r["valid?"] is True


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkReadGaps through the JNI shim and a fake JNIEnv returns what the ctypes binding returns."""
    fj = _rg_fakejvm()
    handle = fj.create()
    try:
        parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, final_reads=True),
                                               torn_pair=s == 2, split_amount=s == 3) for s in (1, 2, 3)]
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_read_gaps(handle, fj.jhistory(h), 0), np.int64)
        g = gpu_ctx.check_read_gaps(h)
        assert v[:9].tolist() == [g[k] for k in ("valid", "n_failures", "n_reads", "n_transfers", "n_explained",
                                                 "n_unexplained", "n_double", "n_undecided", "nodes")]
        assert v[11] == h.n_shards
        for s, q in enumerate(g["shards"]):
            want = [q[f] for f in ("valid", "cause", "n_reads", "n_transfers", "n_explained", "n_undecided")]
            want += q["count_by_kind"] + [q[f] for f in ("nodes", "witness_index", "lower_index", "kind", "key",
                                                         "delta", "transfer_id", "other_index", "n_eligible")]
            assert v[12 + 18 * s: 30 + 18 * s].tolist() == want
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_read_gaps(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])), 0),
                       np.int64)
    finally:
        fj.lib().fj_destroy(handle)
