"""The transfer-placement check on the GPU (K12) against TP_SEARCH, field by field: verdict, per-kind, explained,
undecided and placed counts, node totals, rounds and the witness; K11's gap fields at max_rounds = 1; every error path;
the checker maps and the JNI shim."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from test_monotonic_cpu import inv_r, rd
from test_read_gaps_cpu import REGROUPED, _ones
from test_transfer_lookups_cpu import flat, inv_l, lk, ops_idx, random_tiny, tr
from test_transfer_placement_cpu import CHAINED, LOST, _tp_fakejvm, regrouping, script

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_explained", "n_unexplained", "n_double", "n_lost",
          "n_undecided", "n_placed", "nodes", "rounds", "shards")
GAP_FIELDS = ("n_explained", "n_undecided", "nodes")
MUTATIONS = ("torn_transfer", "torn_pair", "split_amount")


def agree(ctx, h, max_nodes=0, max_rounds=0):
    g = ctx.check_transfer_placement(h, max_nodes, max_rounds)
    o = M.check_transfer_placement(h, M.TP_SEARCH, max_nodes=max_nodes, max_rounds=max_rounds)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    return g


def like_k11(ctx, h):
    """At max_rounds = 1 the gap fields are the read-gap check's."""
    g, k = ctx.check_transfer_placement(h, 0, 1), ctx.check_read_gaps(h)
    for a, b in zip(g["shards"], k["shards"]):
        assert [a[f] for f in GAP_FIELDS] + a["count_by_kind"][:3] == [b[f] for f in GAP_FIELDS] + b["count_by_kind"]


def test_random_tiny_histories(gpu_ctx):
    rng = np.random.default_rng(97)
    kinds = set()
    for i in range(300):
        h = flat(random_tiny(rng)[0])
        kinds.add(agree(gpu_ctx, h, max_nodes=(0, 1, 3)[i % 3], max_rounds=(0, 1, 2)[i % 3 - 1])["shards"][0]["kind"])
        h = flat(regrouping(rng)[0])
        kinds.add(agree(gpu_ctx, h)["shards"][0]["kind"])
        if i % 10 == 0:
            like_k11(gpu_ctx, h)
    assert kinds >= {0, abi.TP_KEY, abi.TP_LOST}, kinds


def test_hand_cases(gpu_ctx):
    assert agree(gpu_ctx, flat(script(CHAINED)[0]))["shards"][0]["kind"] == abi.TP_KEY
    assert agree(gpu_ctx, flat(script(LOST)[0]))["shards"][0]["kind"] == abi.TP_LOST
    assert agree(gpu_ctx, flat(REGROUPED))["shards"][0]["kind"] == abi.TP_KEY
    for mr in (1, 2, 3):
        agree(gpu_ctx, flat(script(CHAINED)[0]), max_rounds=mr)
    for n, shows in ((40, (20, 20)), (70, (35, 35)), (130, (65, 65))):
        agree(gpu_ctx, flat(_ones(n, shows)))
    for mx in (0, 1, 2, 5):
        agree(gpu_ctx, flat(_ones(40, (20, 21))), mx)
    partial = [tr(0, "invoke", 1, 2, 2, 1), inv_r(1, [1, 2]), rd(1, {1: (2, 0), 2: (0, 2)}), inv_r(1, [2]),
               rd(1, {2: (0, 1)})]
    assert agree(gpu_ctx, flat(partial))["shards"][0]["cause"] == abi.CAUSE_PARTIAL_READ


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("variant", ("valid", "stale", "lost_transfer") + MUTATIONS)
def test_c3_size_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, final_reads=True, stale_read=variant == "stale")
    h = synth.generate_ledger_lookups(spec, **({variant: True} if variant in MUTATIONS + ("lost_transfer",) else {}))
    g = agree(gpu_ctx, h)
    like_k11(gpu_ctx, h)
    if variant == "valid":
        assert g["n_unexplained"] == g["n_double"] == g["n_lost"] == 0


def test_crashed_transfers(gpu_ctx):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True))
    g = agree(gpu_ctx, h)
    like_k11(gpu_ctx, h)
    assert g["n_unexplained"] == g["n_double"] == g["n_lost"] == 0
    assert g["n_explained"] >= gpu_ctx.check_read_gaps(h)["n_explained"]


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
        assert g["n_unexplained"] == g["n_double"] == g["n_lost"] == 0


def test_multi_shard(gpu_ctx):
    muts = {2: "torn_transfer", 5: "split_amount", 6: "torn_pair"}
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05,
                                                           final_reads=True), **({muts[s]: True} if s in muts else {}))
             for s in range(1, 9)]
    parts.append(flat(script(CHAINED)[0]))
    parts.append(flat(script(LOST)[0]))
    g = agree(gpu_ctx, H.concat_keys(parts))
    assert len(g["shards"]) == 10 and g["n_lost"] >= 1


@pytest.mark.parametrize("p_info", [0.0, 0.02])
def test_million_op_history(gpu_ctx, p_info):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 1_000_000, 32, 1, p_info=p_info, final_reads=True))
    g = agree(gpu_ctx, h)
    assert g["n_reads"] > 400_000
    assert g["n_unexplained"] == g["n_double"] == g["n_lost"] == 0


def test_errors_leave_the_context_usable(gpu_ctx):
    ok = [tr(0, "invoke", 1, 2, 1, 1), tr(0, "ok", 1, 2, 1, 1)]
    lost = flat(script(LOST)[0])

    def raises(ops, match, mutate=None):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(NativeError, match=match):
            gpu_ctx.check_transfer_placement(h)
        assert agree(gpu_ctx, lost)["valid"] == H.INVALID

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", -1, 2, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, 0))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises(ok + [inv_l(1), lk(1, [(1, 1, 2, 1)])], "multiple of 5", lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "multiple of 3", lambda h: h.payload_len.__setitem__(1, 5))
    ch = H.as_c_history(flat(ok))
    shards, res = (abi.CTpShard * 1)(), abi.CTpResult()
    assert native.lib().jtb_check_transfer_placement(gpu_ctx._h, C.addressof(ch), 0, 0, 1, C.addressof(shards),
                                                     C.addressof(res)) < 0
    assert "reserved" in gpu_ctx._err()
    assert agree(gpu_ctx, lost)["valid"] == H.INVALID


def test_checker_result_map(gpu_ctx):
    r = checker.transfer_placement_checker(ctx=gpu_ctx).check({}, ops_idx(script(LOST)[0]))
    assert r["valid?"] is False and r["errors"] == {"lost": 1} and r["op"] == {"index": 6}
    comp = checker.ledger_checker(ctx=gpu_ctx, linear=False, transfer_placement=True).check(
        {"accounts": [1, 2]}, ops_idx(script(CHAINED)[0]))
    assert comp["transfer-placement"]["valid?"] is False and comp["valid?"] is False
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 600, 8, s, tau_think_ns=5e6, final_reads=True))
             for s in (1, 2, 3)]
    r = checker.independent_checker(checker.transfer_placement_checker(ctx=gpu_ctx)).check({}, H.concat_keys(parts))
    assert r["valid?"] is True


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkTransferPlacement through the JNI shim and a fake JNIEnv returns what ctypes returns."""
    fj = _tp_fakejvm()
    handle = fj.create()
    try:
        parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, final_reads=True),
                                               torn_pair=s == 2, split_amount=s == 3) for s in (1, 2, 3)]
        parts.append(flat(script(LOST)[0]))
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_transfer_placement(handle, fj.jhistory(h), 0, 0), np.int64)
        g = gpu_ctx.check_transfer_placement(h)
        assert v[:12].tolist() == [g[k] for k in ("valid", "n_failures", "n_reads", "n_transfers", "n_explained",
                                                  "n_unexplained", "n_double", "n_lost", "n_undecided", "n_placed",
                                                  "nodes", "rounds")]
        assert v[14] == h.n_shards
        for s, q in enumerate(g["shards"]):
            want = [q[f] for f in ("valid", "cause", "n_reads", "n_transfers", "n_explained", "n_undecided")]
            want += q["count_by_kind"] + [q[f] for f in ("n_placed", "nodes", "rounds", "witness_index",
                                                         "lower_index", "kind", "key", "round", "delta",
                                                         "transfer_id", "other_index", "n_eligible")]
            assert v[15 + 22 * s: 37 + 22 * s].tolist() == want
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_transfer_placement(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])),
                                                            0, 0), np.int64)
    finally:
        fj.lib().fj_destroy(handle)
