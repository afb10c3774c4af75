"""The counter-bounds check without a GPU: hand KATs in ledger form against both CPU deciders, their soundness against a
brute-force search for a serial explanation, the two deciders against each other, the multi-transfer guard, the
synthetic lost / duplicated transfer histories and the ABI images of the new structs."""
import ctypes
import hashlib

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, synth
from jepsen_tigerbeetle_b200 import history as H
from test_monotonic_cpu import flat, inv_r, rd, tr

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_violations", "shards")


def both(h):
    """CB_LITERAL and CB_SWEEP, which must agree field by field; returns the first."""
    lit = M.check_counter_bounds(h, M.CB_LITERAL)
    sw = M.check_counter_bounds(h, M.CB_SWEEP)
    assert {k: lit[k] for k in FIELDS} == {k: sw[k] for k in FIELDS}, (lit, sw)
    return lit


def shard(h):
    return both(h)["shards"][0]


def witness(s):
    return (s["witness_index"], s["witness_key"], s["kind"], s["value"], s["bound"], s["culprit_index"])


def final(op):
    return dict(op, **{"final?": True})


SEEN = {1: (1, 0), 2: (0, 1)}     # a read that saw one transfer 1 -> 2 of amount 1
UNSEEN = {1: (0, 0), 2: (0, 0)}


# ---- KATs -----------------------------------------------------------------------------------------------------
def test_b42_is_below():
    """SURVEY B42: the read misses the second transfer, which completed before it was invoked (K7 passes it)."""
    ops = [tr(0, "invoke", 1, 2, 3), tr(0, "ok", 1, 2, 3), tr(0, "invoke", 2, 3, 1), tr(0, "ok", 2, 3, 1),
           inv_r(0, [1, 2, 3]), rd(0, {1: (3, 0), 2: (0, 3), 3: (0, 0)})]
    s = shard(flat(ops))
    assert s["valid"] == H.INVALID
    # key 4 = [2, "debits-posted"]: value 0, L = 1, the transfer completing at :index 3 is missing
    assert witness(s) == (5, H.counter_key(2, 0), abi.CB_BELOW, 0, 1, 3)
    assert (s["n_below"], s["n_above"], s["n_reads"], s["n_transfers"], s["n_keys"]) == (2, 0, 1, 2, 6)


def test_b46_concurrent_transfer_unseen_is_valid():
    ops = [tr(0, "invoke", 1, 2, 1), inv_r(1, [1, 2]), rd(1, UNSEEN), tr(0, "ok", 1, 2, 1)]
    assert shard(flat(ops))["valid"] == H.VALID


def test_concurrent_transfer_seen_is_valid():
    ops = [tr(0, "invoke", 1, 2, 1), inv_r(1, [1, 2]), rd(1, SEEN), tr(0, "ok", 1, 2, 1)]
    assert shard(flat(ops))["valid"] == H.VALID


def test_transfer_invoked_after_the_read_completed_is_above():
    ops = [inv_r(1, [1, 2]), rd(1, SEEN), tr(0, "invoke", 1, 2, 1), tr(0, "ok", 1, 2, 1)]
    s = shard(flat(ops))
    assert witness(s) == (1, H.counter_key(1, 0), abi.CB_ABOVE, 1, 0, -1)
    assert (s["n_below"], s["n_above"]) == (0, 2)


def test_seen_failed_transfer_is_above():
    ops = [tr(0, "invoke", 1, 2, 1), tr(0, "fail", 1, 2, 1), inv_r(1, [1, 2]), rd(1, SEEN)]
    s = shard(flat(ops))
    assert witness(s) == (3, H.counter_key(1, 0), abi.CB_ABOVE, 1, 0, -1)
    assert s["n_transfers"] == 0


@pytest.mark.parametrize("seen", [False, True])
def test_info_transfer(seen):
    before = [tr(0, "invoke", 1, 2, 1), tr(0, "info", 1, 2, 1), inv_r(1, [1, 2]), rd(1, SEEN if seen else UNSEEN)]
    assert shard(flat(before))["valid"] == H.VALID
    after = [inv_r(1, [1, 2]), rd(1, SEEN if seen else UNSEEN), tr(0, "invoke", 1, 2, 1), tr(0, "info", 1, 2, 1)]
    s = shard(flat(after))
    if seen:   # invoked after the read completed: it cannot be inside the read
        assert witness(s) == (1, H.counter_key(1, 0), abi.CB_ABOVE, 1, 0, -1)
    else:
        assert s["valid"] == H.VALID


def test_never_completed_transfer_counts_in_u_only():
    for vals in ({1: (4, 0), 2: (0, 4)}, UNSEEN):
        s = shard(flat([tr(0, "invoke", 1, 2, 4), inv_r(1, [1, 2]), rd(1, vals)]))
        assert (s["valid"], s["n_transfers"]) == (H.VALID, 1)
    # the same transfer completed :ok before the read: now L holds it too
    s = shard(flat([tr(0, "invoke", 1, 2, 4), tr(0, "ok", 1, 2, 4), inv_r(1, [1, 2]), rd(1, UNSEEN)]))
    assert witness(s) == (3, H.counter_key(1, 0), abi.CB_BELOW, 0, 4, 1)


def test_untouched_key_must_read_zero():
    assert shard(flat([inv_r(0, [1]), rd(0, {1: (0, 0)})]))["valid"] == H.VALID
    s = shard(flat([inv_r(0, [1]), rd(0, {1: (0, 2)})]))
    assert witness(s) == (1, H.counter_key(1, 1), abi.CB_ABOVE, 2, 0, -1)
    s = shard(flat([inv_r(0, [1]), rd(0, {1: (-1, 0)})]))   # below an empty L: no culprit
    assert witness(s) == (1, H.counter_key(1, 0), abi.CB_BELOW, -1, 0, -1)


def test_partial_reads_are_decided():
    """K7's partial-read KAT (UNKNOWN there): every bound is per (read, key), so it is decided here."""
    ops = [inv_r(0, [1, 2]), inv_r(1, [2, 3]), inv_r(2, [3, 1]),
           rd(0, {1: (1, 1), 2: (0, 0)}), rd(1, {2: (1, 1), 3: (0, 0)}), rd(2, {3: (1, 1), 1: (0, 0)})]
    s = shard(flat(ops))
    assert witness(s) == (3, H.counter_key(1, 0), abi.CB_ABOVE, 1, 0, -1)
    assert (s["n_above"], s["n_keys"]) == (6, 6)
    # with the transfers that explain them the same partial reads are VALID
    ops = [tr(3, "invoke", 1, 1, 1), tr(4, "invoke", 2, 2, 1), tr(5, "invoke", 3, 3, 1)] + ops
    assert shard(flat(ops))["valid"] == H.VALID


def test_lost_transfer_seen_by_a_final_read():
    ops = [tr(0, "invoke", 1, 2, 5), tr(0, "ok", 1, 2, 5), tr(0, "invoke", 2, 1, 2), tr(0, "ok", 2, 1, 2),
           inv_r(1, [1, 2]), final(rd(1, {1: (0, 2), 2: (2, 0)}))]
    s = shard(flat(ops))
    assert witness(s) == (5, H.counter_key(1, 0), abi.CB_BELOW, 0, 5, 1)
    assert (s["n_below"], s["n_above"]) == (2, 0)


def test_errors():
    h = flat([tr(0, "invoke", 1, 2, -1), tr(0, "ok", 1, 2, -1)])
    with pytest.raises(RuntimeError, match="negative amount"):
        M.check_counter_bounds(h)
    h = flat([tr(0, "invoke", 1, 1 << 30, 1)])
    with pytest.raises(RuntimeError, match="outside"):
        M.check_counter_bounds(h)
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload_len[1] = 5
    with pytest.raises(RuntimeError, match="payload"):
        M.check_counter_bounds(h)
    with pytest.raises(RuntimeError, match="reserved"):
        M.check_counter_bounds(flat([inv_r(0, [1]), rd(0, {1: (0, 0)})]), flags=1)


# ---- soundness: a serial explanation means VALID ----------------------------------------------------------------
def random_tiny(rng):
    """A random tiny ledger history (<= 3 accounts, <= 8 ops) with :ok, :info, :fail and never-completed transfers.
    Transfers take effect at their completion (an :info one half the time); reads return the counters at their
    completion, sometimes with one key off by one.  Returns (op maps, op records for the brute force)."""
    n_acct, n_proc, n_ops = int(rng.integers(1, 4)), int(rng.integers(1, 4)), int(rng.integers(1, 9))
    deb, cred = [0] * n_acct, [0] * n_acct
    ops, recs, open_ops, started = [], [], {}, 0
    while started < n_ops or (open_ops and rng.random() < 0.7):
        p = int(rng.integers(0, n_proc))
        if p in open_ops:
            r = open_ops.pop(p)
            r["comp"] = len(ops)
            if r["kind"] == "t":
                fate = str(rng.choice(["ok", "ok", "info", "fail"]))
                r["fate"] = fate
                if fate == "ok" or (fate == "info" and rng.random() < 0.5):
                    deb[r["b"] - 1] += r["a"]
                    cred[r["c"] - 1] += r["a"]
                ops.append(tr(p, fate, r["b"], r["c"], r["a"]))
            else:
                d, c = list(deb), list(cred)
                if rng.random() < 0.3:
                    j = int(rng.integers(0, n_acct))
                    if rng.random() < 0.5:
                        d[j] += int(rng.choice([-1, 1]))
                    else:
                        c[j] += int(rng.choice([-1, 1]))
                r["fate"] = "ok" if rng.random() < 0.9 else "info"
                r["values"] = {H.counter_key(a + 1, 0): d[a] for a in range(n_acct)}
                r["values"].update({H.counter_key(a + 1, 1): c[a] for a in range(n_acct)})
                ops.append(rd(p, {a + 1: (d[a], c[a]) for a in range(n_acct)}, r["fate"]))
        elif started < n_ops:
            started += 1
            if rng.random() < 0.5:
                r = {"kind": "r", "inv": len(ops), "comp": None, "fate": None}
                ops.append(inv_r(p, list(range(1, n_acct + 1))))
            else:
                b = int(rng.integers(1, n_acct + 1))
                c = int(rng.integers(1, n_acct + 1))
                r = {"kind": "t", "inv": len(ops), "comp": None, "fate": None, "a": int(rng.integers(0, 3)),
                     "b": b, "c": c}
                ops.append(tr(p, "invoke", b, c, r["a"]))
            open_ops[p] = r
            recs.append(r)
    return ops, recs


def explainable(recs) -> bool:
    """Is there a serial order of the :ok reads, the :ok transfers and some of the :info / never-completed transfers
    that respects real time, in which every :ok read returns the counters of the transfers before it?"""
    must = [r for r in recs if (r["kind"] == "r" and r["fate"] == "ok") or (r["kind"] == "t" and r["fate"] == "ok")]
    maybe = [r for r in recs if r["kind"] == "t" and r["fate"] in ("info", None)]
    for pick in range(1 << len(maybe)):
        ops = must + [m for i, m in enumerate(maybe) if pick >> i & 1]
        n = len(ops)
        pred = [sum(1 << j for j, y in enumerate(ops) if y["comp"] is not None and y["comp"] < x["inv"])
                for x in ops]
        reach = {0}
        for mask in range(1 << n):
            if mask not in reach:
                continue
            cnt: dict[int, int] = {}
            for j, y in enumerate(ops):
                if mask >> j & 1 and y["kind"] == "t":
                    cnt[H.counter_key(y["b"], 0)] = cnt.get(H.counter_key(y["b"], 0), 0) + y["a"]
                    cnt[H.counter_key(y["c"], 1)] = cnt.get(H.counter_key(y["c"], 1), 0) + y["a"]
            for j, x in enumerate(ops):
                if mask >> j & 1 or pred[j] & ~mask:
                    continue
                if x["kind"] == "r" and any(cnt.get(k, 0) != v for k, v in x["values"].items()):
                    continue
                reach.add(mask | 1 << j)
        if (1 << n) - 1 in reach:
            return True
    return False


def test_sound_against_brute_force():
    rng = np.random.default_rng(21)
    verdicts = {H.VALID: 0, H.INVALID: 0}
    explained = 0
    for _ in range(2000):
        ops, recs = random_tiny(rng)
        v = both(flat(ops))["valid"]
        verdicts[v] += 1
        if explainable(recs):
            explained += 1
            assert v == H.VALID, ops
    assert verdicts[H.VALID] > 200 and verdicts[H.INVALID] > 200, verdicts
    assert explained > 200


# ---- the two deciders agree on C3-size synthetic histories ------------------------------------------------------
@pytest.mark.parametrize("variant", ["valid", "stale", "fractured", "lost", "duplicated", "info"])
def test_oracles_agree_on_c3_size(variant):
    spec = synth.SynthSpec("bank", 10000, 32, 2, stale_read=variant == "stale", final_reads=True,
                           p_info=0.02 if variant == "info" else 0.0)
    h = synth.generate_ledger_counters(spec, fractured=variant == "fractured", lost_transfer=variant == "lost",
                                       duplicated_transfer=variant == "duplicated")
    r = both(h)
    assert r["n_reads"] > 4000
    if variant in ("valid", "info"):
        assert r["valid"] == H.VALID
    if variant in ("lost", "duplicated"):
        assert r["shards"][0]["kind"] == (abi.CB_BELOW if variant == "lost" else abi.CB_ABOVE)


def test_oracles_agree_on_many_keys():
    parts = [synth.generate_ledger_counters(synth.SynthSpec("bank", 800, 8, s, tau_think_ns=5e6, final_reads=True),
                                            lost_transfer=s % 3 == 0, duplicated_transfer=s % 3 == 1)
             for s in range(1, 10)]
    r = both(H.concat_keys(parts))
    assert [s["valid"] for s in r["shards"]] == [H.INVALID if s % 3 != 2 else H.VALID for s in range(1, 10)]


# ---- flattener and checker guard --------------------------------------------------------------------------------
def test_multi_transfer_txns_are_counted_and_refused():
    two = [["t", 0, {"debit-acct": 1, "credit-acct": 2, "amount": 1}],
           ["t", 1, {"debit-acct": 2, "credit-acct": 1, "amount": 1}]]
    ops = [{"type": "invoke", "process": 0, "f": "txn", "value": two},
           {"type": "ok", "process": 0, "f": "txn", "value": two}, inv_r(1, [1, 2]), rd(1, UNSEEN)]
    one = flat([tr(0, "invoke", 1, 2, 1), tr(0, "ok", 1, 2, 1), inv_r(1, [1, 2]), rd(1, UNSEEN)])
    h = flat(ops)
    assert h.meta["multi_transfer_txns"] == 1 and one.meta["multi_transfer_txns"] == 0
    for name in ("type", "f", "process", "index", "a", "b", "c", "payload_off", "payload_len", "payload"):
        assert np.array_equal(getattr(h, name), getattr(one, name)), name   # only the first [:t ...] is kept
    r = checker.check_safe(checker.counter_bounds_checker(), {}, [dict(o, index=i) for i, o in enumerate(ops)])
    assert r["valid?"] == "unknown" and "more than one" in r["error"]


# ---- synthetic histories ----------------------------------------------------------------------------------------
def _digest(h) -> str:
    m = hashlib.sha256()
    for n in ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_off", "payload_len",
              "payload", "shard_off", "key_ids"):
        a = np.ascontiguousarray(getattr(h, n))
        m.update(n.encode())
        m.update(str(a.dtype).encode())
        m.update(a.tobytes())
    return m.hexdigest()


@pytest.mark.parametrize("spec,kw,digest", [
    (synth.SynthSpec("bank", 3000, 16, 5, p_info=0.05, stale_read=True), {},
     "f5ccd4f7b64a016cc1d4e8d0f3fe6e3d370913fc3395861e062f01ccb1ee8ca7"),
    (synth.SynthSpec("bank", 2000, 8, 2, n_keys=3), {"fractured": True},
     "f260a565bcc1cf8a43d0226983e3a7bc25d64121c11d59f7636157102c95ae43"),
    (synth.SynthSpec("bank", 1000, 8, 1), {}, "424fce67b31cec6c0e3ae54c270650989a9d8e761aebbb70236463ed4a30564d"),
])
def test_default_ledger_counter_output_is_unchanged(spec, kw, digest):
    """Digests of generate_ledger_counters output taken before lost / duplicated transfers and final reads existed."""
    h = synth.generate_ledger_counters(spec, **kw)
    assert _digest(h) == digest
    assert "lost_op_index" not in h.meta and "duplicated_op_index" not in h.meta


@pytest.mark.parametrize("mutation", ["lost_transfer", "duplicated_transfer"])
def test_lost_and_duplicated_transfers(mutation):
    spec = synth.SynthSpec("bank", 1500, 16, 3, final_reads=True)
    base = synth.generate_ledger_counters(spec)
    h = synth.generate_ledger_counters(spec, **{mutation: True})
    key = "lost_op_index" if mutation == "lost_transfer" else "duplicated_op_index"
    assert h.meta[key] >= 0
    for name in ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_off", "payload_len"):
        assert np.array_equal(getattr(h, name), getattr(base, name)), name
    assert not np.array_equal(h.payload, base.payload)
    assert both(base)["valid"] == H.VALID
    r = both(h)
    assert r["valid"] == H.INVALID
    s = r["shards"][0]
    assert (s["kind"], s["n_below"] > 0, s["n_above"] > 0) == (
        (abi.CB_BELOW, True, False) if mutation == "lost_transfer" else (abi.CB_ABOVE, False, True))


def test_final_reads_return_the_final_counters():
    spec = synth.SynthSpec("bank", 600, 8, 4, final_reads=True, p_info=0.05)
    h = synth.generate_ledger_counters(spec)
    fin = np.nonzero((h.flags & H.FLAG_FINAL) & (h.type == H.T_OK))[0]
    assert len(fin) == 1
    tri = h.payload[h.payload_off[fin[0]]:h.payload_off[fin[0]] + h.payload_len[fin[0]]].reshape(-1, 3)
    assert tri[:, 1].sum() > 0 and tri[:, 1][0::2].sum() == tri[:, 1][1::2].sum()   # debits total = credits total
    assert both(h)["valid"] == H.VALID


# ---- ABI ------------------------------------------------------------------------------------------------------
def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(11) == ctypes.sizeof(abi.CCbShard) == 64
    assert lib.jtb_struct_size(12) == ctypes.sizeof(abi.CCbResult) == 48
