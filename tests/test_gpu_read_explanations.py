"""The read-explanation check on the GPU (K10) against RX_SEARCH, field by field: verdict, per-kind, explained and
undecided counts, node totals and the witness (op, kind, key, |must|, |may|, value, must sum); every error path; the
checker maps and the JNI shim."""
import ctypes as C

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, native, synth
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError
from test_monotonic_cpu import inv_r, rd
from test_read_explanations_cpu import TORN_PAIR, _rx_fakejvm
from test_transfer_lookups_cpu import flat, inv_l, lk, ops_idx, random_tiny, tr

pytestmark = pytest.mark.gpu

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_explained", "n_unexplained", "n_undecided", "nodes",
          "shards")
MUTATIONS = ("torn_transfer", "torn_pair", "split_amount")


def agree(ctx, h, max_nodes=0):
    g = ctx.check_read_explanations(h, max_nodes)
    o = M.check_read_explanations(h, M.RX_SEARCH, max_nodes=max_nodes)
    assert {k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS}
    return g


def test_random_tiny_histories(gpu_ctx):
    rng = np.random.default_rng(47)
    kinds = set()
    for i in range(400):
        g = agree(gpu_ctx, flat(random_tiny(rng)[0]), max_nodes=(0, 1, 3)[i % 3])
        kinds.add(g["shards"][0]["kind"])
    assert kinds >= {0, abi.RX_KEY}, kinds


def test_hand_cases(gpu_ctx):
    assert agree(gpu_ctx, flat(TORN_PAIR))["shards"][0]["kind"] == abi.RX_JOINT
    for n in (40, 70):   # decided by the search / more than 64 free candidates
        ops = [tr(p, "invoke", 1, 2, 1, p + 1) for p in range(n)] + [inv_r(n, [1, 2]), rd(n, {1: (20, 0), 2: (0, 20)})]
        agree(gpu_ctx, flat(ops + [tr(p, "ok", 1, 2, 1, p + 1) for p in range(n)]))
    ops = [tr(p, "invoke", 1, 2, 3 if p < 6 else 2, p + 1) for p in range(12)]
    ops += [inv_r(12, [1, 2]), rd(12, {1: (1, 0), 2: (0, 1)})] + [tr(p, "ok", 1, 2, 3 if p < 6 else 2, p + 1)
                                                                   for p in range(12)]
    for mx in (0, 1, 2, 5):
        agree(gpu_ctx, flat(ops), mx)


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("variant", ("valid", "stale", "fractured", "lost_transfer") + MUTATIONS)
def test_c3_size_histories(gpu_ctx, seed, variant):
    spec = synth.SynthSpec("bank", 10000, 32, seed, final_reads=True, stale_read=variant == "stale")
    if variant == "fractured":   # the counter form's fractured read on the lookups form's events
        c = synth.generate_ledger_counters(spec, fractured=True)
        h = synth.generate_ledger_lookups(spec)
        reads = np.nonzero((h.f == H.F_READ) & (h.type == H.T_OK))[0]
        creads = np.nonzero((c.f == H.F_READ) & (c.type == H.T_OK))[0]
        for e, ce in zip(reads, creads):
            h.payload[h.payload_off[e]:h.payload_off[e] + h.payload_len[e]] = \
                c.payload[c.payload_off[ce]:c.payload_off[ce] + c.payload_len[ce]]
    else:
        h = synth.generate_ledger_lookups(spec, **({variant: True} if variant in MUTATIONS + ("lost_transfer",) else {}))
    g = agree(gpu_ctx, h)
    if variant in MUTATIONS + ("lost_transfer",):
        assert g["valid"] == H.INVALID
    if variant == "valid":
        assert g["n_unexplained"] == 0


def test_crashed_transfers(gpu_ctx):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True))
    assert np.count_nonzero(h.type == H.T_INFO) > 100
    g = agree(gpu_ctx, h)
    assert g["n_unexplained"] == 0 and g["n_explained"] > 0.9 * g["n_reads"]


def test_mid_history_lookups(gpu_ctx):
    spec = synth.SynthSpec("bank", 600, 8, 2, p_info=0.05, final_reads=True)
    for kw in ({}, {"lost_transfer": True}, {"torn_pair": True}):
        agree(gpu_ctx, synth.generate_ledger_lookups(spec, p_lookup=0.05, **kw))


@pytest.mark.parametrize("kw", [{}, {"torn_pair": True}])
def test_64_accounts(gpu_ctx, kw):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, p_info=0.02,
                                                      final_reads=True), **kw)
    g = agree(gpu_ctx, h)
    assert g["valid"] == H.INVALID if kw else g["n_unexplained"] == 0


def test_multi_shard(gpu_ctx):
    muts = {2: "torn_transfer", 5: "split_amount", 6: "torn_pair"}
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05,
                                                           final_reads=True), **({muts[s]: True} if s in muts else {}))
             for s in range(1, 9)]
    g = agree(gpu_ctx, H.concat_keys(parts))
    assert [s["valid"] == H.INVALID for s in g["shards"]] == [s in muts for s in range(1, 9)]


@pytest.mark.parametrize("kw", [{}, {"torn_pair": True}])
def test_million_op_history(gpu_ctx, kw):
    h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 1_000_000, 32, 1, final_reads=True), **kw)
    g = agree(gpu_ctx, h)
    assert g["n_reads"] > 400_000 and (g["valid"] == H.INVALID) == bool(kw)


def test_errors_leave_the_context_usable(gpu_ctx):
    ok = [tr(0, "invoke", 1, 2, 1, 1), tr(0, "ok", 1, 2, 1, 1)]

    def raises(ops, match, mutate=None):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(NativeError, match=match):
            gpu_ctx.check_read_explanations(h)
        assert agree(gpu_ctx, flat(TORN_PAIR))["valid"] == H.INVALID

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", -1, 2, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, 0))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises(ok + [inv_l(1), lk(1, [(1, 1, 2, 1)])], "multiple of 5", lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "multiple of 3", lambda h: h.payload_len.__setitem__(1, 5))
    h = flat(ok)
    ch = H.as_c_history(h)
    shards, res = (abi.CRxShard * 1)(), abi.CRxResult()
    assert native.lib().jtb_check_read_explanations(gpu_ctx._h, C.addressof(ch), 0, 1, C.addressof(shards),
                                                    C.addressof(res)) < 0
    assert "reserved" in gpu_ctx._err()
    assert agree(gpu_ctx, flat(TORN_PAIR))["valid"] == H.INVALID


def test_checker_result_map(gpu_ctx):
    r = checker.read_explanation_checker(ctx=gpu_ctx).check({}, ops_idx(TORN_PAIR))
    assert r["valid?"] is False and r["errors"] == {"joint": 1} and r["op"] == {"index": 3}
    comp = checker.ledger_checker(ctx=gpu_ctx, linear=False, read_explanations=True).check({"accounts": [1, 2, 3, 4]},
                                                                                            ops_idx(TORN_PAIR))
    assert comp["read-explanations"]["valid?"] is False and comp["valid?"] is False
    parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 600, 8, s, tau_think_ns=5e6, final_reads=True),
                                           torn_pair=s == 2) for s in (1, 2, 3)]
    h = H.concat_keys(parts)
    r = checker.independent_checker(checker.read_explanation_checker(ctx=gpu_ctx)).check({}, h)
    assert r["valid?"] is False and int(h.key_ids[1]) in r["failures"]


def test_jni_shim_equals_ctypes(gpu_ctx):
    """jtb.Native.checkReadExplanations through the JNI shim and a fake JNIEnv returns what the ctypes binding
    returns."""
    fj = _rx_fakejvm()
    handle = fj.create()
    try:
        parts = [synth.generate_ledger_lookups(synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, final_reads=True),
                                               torn_pair=s == 2, split_amount=s == 3) for s in (1, 2, 3)]
        h = H.concat_keys(parts)
        v = fj._result(fj.lib().fj_check_read_explanations(handle, fj.jhistory(h), 0), np.int64)
        g = gpu_ctx.check_read_explanations(h)
        assert v[:8].tolist() == [g[k] for k in ("valid", "n_failures", "n_reads", "n_transfers", "n_explained",
                                                 "n_unexplained", "n_undecided", "nodes")]
        assert v[10] == h.n_shards
        for s, q in enumerate(g["shards"]):
            want = [q[f] for f in ("valid", "n_reads", "n_transfers", "witness_index", "n_explained", "n_undecided")]
            want += q["count_by_kind"] + [q[f] for f in ("nodes", "kind", "key", "n_must", "n_may", "value",
                                                         "must_sum")]
            assert v[11 + 15 * s: 26 + 15 * s].tolist() == want
        with pytest.raises(fj.JavaException, match="negative amount"):
            fj._result(fj.lib().fj_check_read_explanations(handle, fj.jhistory(flat([tr(0, "invoke", 1, 2, -5, 1)])),
                                                           0), np.int64)
    finally:
        fj.lib().fj_destroy(handle)
