"""The monotonic-key check without a GPU: hand KATs in ledger form against both CPU deciders, the two deciders against
each other on random full-key histories, the ledger-counters flattener, the synthetic ledger-counter generator and
the ABI images of the new structs."""
import ctypes

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, synth
from jepsen_tigerbeetle_b200 import history as H

def _acct(d, c):
    return {"debits-posted": d, "credits-posted": c}


def rd(p, accts, typ="ok"):
    """A ledger :r txn of process p; accts = {account: (debits, credits) | None}."""
    return {"type": typ, "process": p, "f": "txn",
            "value": [["r", a, None if v is None else _acct(*v)] for a, v in accts.items()]}


def inv_r(p, accts):
    return {"type": "invoke", "process": p, "f": "txn", "value": [["r", a, None] for a in accts]}


def tr(p, typ, d, c, amount):
    return {"type": typ, "process": p, "f": "txn",
            "value": [["t", 0, {"debit-acct": d, "credit-acct": c, "amount": amount}]]}


def flat(ops):
    return H.flatten_ops([dict(o, index=i) for i, o in enumerate(ops)], "ledger-counters")


def both(h, realtime=True, decide_partial=False):
    g = M.check_monotonic_keys(h, M.MONO_GRAPH, realtime, decide_partial)
    p = M.check_monotonic_keys(h, M.MONO_PAIRS, realtime, decide_partial)
    return g, p


# ---- KATs -----------------------------------------------------------------------------------------------------
def test_crossed_pair_is_invalid():
    # two concurrent reads: one saw account 1 debited and account 2 not, the other the reverse
    h = flat([inv_r(0, [1, 2]), inv_r(1, [1, 2]),
              rd(0, {1: (1, 0), 2: (0, 0)}), rd(1, {1: (0, 0), 2: (1, 0)})])
    for rt in (True, False):
        g, p = both(h, rt)
        assert g["shards"] == p["shards"]
        s = g["shards"][0]
        assert s["valid"] == H.INVALID and s["n_reads"] == 2 and s["n_keys"] == 4
        assert (s["witness_index"], s["partner_index"]) == (3, 2)
        # partner -> witness on account 2's debits, witness -> partner on account 1's debits
        assert s["edges"] == [(abi.MONO_EDGE_MONOTONIC, 4, 0, 1), (abi.MONO_EDGE_MONOTONIC, 2, 0, 1)]


def test_realtime_stale_read():
    # a read that starts after another one finished sees an older debits-posted
    ops = [inv_r(0, [1]), rd(0, {1: (2, 0)}), inv_r(1, [1]), rd(1, {1: (1, 0)})]
    h = flat(ops)
    g, p = both(h, True)
    assert g["shards"] == p["shards"]
    s = g["shards"][0]
    assert (s["valid"], s["witness_index"], s["partner_index"]) == (H.INVALID, 3, 1)
    assert s["edges"] == [(abi.MONO_EDGE_REALTIME, -1, 1, 2), (abi.MONO_EDGE_MONOTONIC, 2, 1, 2)]
    g, p = both(h, False)
    assert g["valid"] == p["valid"] == H.VALID


@pytest.mark.parametrize("ordered", [False, True])
def test_equal_counters_are_valid(ordered):
    same = {1: (3, 1), 2: (1, 3)}
    ops = ([inv_r(0, [1, 2]), rd(0, same), inv_r(1, [1, 2]), rd(1, same)] if ordered else
           [inv_r(0, [1, 2]), inv_r(1, [1, 2]), rd(0, same), rd(1, same)])
    for rt in (True, False):
        g, p = both(flat(ops), rt)
        assert g["valid"] == p["valid"] == H.VALID


def test_b42_is_valid_here():
    """SURVEY B42 (a stale read that preserves the total; not linearizable) has one read: no cycle is possible, so
    this check is weaker than :linear."""
    ops = [tr(0, "invoke", 1, 2, 3), tr(0, "ok", 1, 2, 3), tr(0, "invoke", 2, 3, 1), tr(0, "ok", 2, 3, 1),
           inv_r(0, [1, 2, 3]), rd(0, {1: (3, 0), 2: (0, 3), 3: (0, 0)})]
    g, p = both(flat(ops))
    assert g["valid"] == p["valid"] == H.VALID
    assert g["shards"][0]["n_reads"] == 1


def test_partial_read_three_cycle():
    # r{1,2} -> s{2,3} -> t{3,1} -> r, and no two of them form a 2-cycle
    ops = [inv_r(0, [1, 2]), inv_r(1, [2, 3]), inv_r(2, [3, 1]),
           rd(0, {1: (1, 1), 2: (0, 0)}), rd(1, {2: (1, 1), 3: (0, 0)}), rd(2, {3: (1, 1), 1: (0, 0)})]
    h = flat(ops)
    g, p = both(h)
    for r in (g, p):
        s = r["shards"][0]
        assert (s["valid"], s["cause"], s["witness_index"]) == (H.UNKNOWN, abi.CAUSE_PARTIAL_READ, -1)
    g, p = both(h, decide_partial=True)
    assert g["valid"] == H.INVALID and g["shards"][0]["witness_index"] == 5
    assert p["valid"] == H.VALID


def test_transfers_info_and_failed_ops_are_not_nodes():
    ops = [inv_r(0, [1]), tr(1, "invoke", 1, 2, 1), rd(0, {1: (0, 0)}, typ="info"), tr(1, "info", 1, 2, 1),
           inv_r(2, [1]), rd(2, {1: (5, 0)}, typ="fail"), inv_r(3, [1]), rd(3, {1: (1, 0)})]
    g, _ = both(flat(ops))
    assert g["valid"] == H.VALID and g["n_reads"] == 1


def test_malformed_payload_is_an_error():
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload_len[1] = 5
    with pytest.raises(RuntimeError, match="payload"):
        M.check_monotonic_keys(h)
    h = flat([inv_r(0, [1]), rd(0, {1: (1, 0)})])
    h.payload[3] = h.payload[0]   # the same key twice
    with pytest.raises(RuntimeError, match="twice"):
        M.check_monotonic_keys(h)


# ---- the two deciders agree on random full-key histories ----------------------------------------------------------
def random_history(rng, n_ops=None):
    """A random ledger-counter history: n_proc clients, every read observes every account; the counters a read sees are
    the true ones, sometimes an older snapshot of one account or of all of them."""
    n_acct = int(rng.integers(1, 4))
    n_proc = int(rng.integers(1, 5))
    n_ops = n_ops or int(rng.integers(2, 14))
    deb = [0] * n_acct
    cred = [0] * n_acct
    hist = [(tuple(deb), tuple(cred))]
    ops, open_ops = [], {}
    for _ in range(n_ops * 2):
        p = int(rng.integers(0, n_proc))
        if p in open_ops:
            kind = open_ops.pop(p)
            if kind == "t":
                a, b = (int(x) for x in rng.choice(n_acct, 2, replace=False)) if n_acct > 1 else (0, 0)
                if n_acct > 1:
                    deb[a] += 1
                    cred[b] += 1
                    hist.append((tuple(deb), tuple(cred)))
                ops.append(tr(p, "ok", a + 1, b + 1, 1))
            else:
                d, c = hist[-1]
                u = rng.random()
                if u < 0.25:
                    d, c = hist[int(rng.integers(0, len(hist)))]
                elif u < 0.4:
                    j = int(rng.integers(0, n_acct))
                    od, oc = hist[int(rng.integers(0, len(hist)))]
                    d = d[:j] + (od[j],) + d[j + 1:]
                    c = c[:j] + (oc[j],) + c[j + 1:]
                typ = "ok" if rng.random() < 0.9 else "info"
                ops.append(rd(p, {j + 1: (d[j], c[j]) for j in range(n_acct)}, typ))
        else:
            if rng.random() < 0.5:
                open_ops[p] = "r"
                ops.append(inv_r(p, list(range(1, n_acct + 1))))
            else:
                open_ops[p] = "t"
                ops.append(tr(p, "invoke", 1, 2, 1))
    return flat(ops)


@pytest.mark.parametrize("realtime", [True, False])
def test_graph_equals_pairs_on_random_full_key_histories(realtime):
    rng = np.random.default_rng(7 if realtime else 8)
    n_invalid = 0
    for _ in range(1000):
        h = random_history(rng)
        g, p = both(h, realtime)
        assert g["shards"] == p["shards"], (g, p)
        n_invalid += g["valid"] == H.INVALID
    assert 20 < n_invalid < 980   # both verdicts are represented


# ---- flattener ------------------------------------------------------------------------------------------------
def test_flatten_key_encoding_and_int64_values():
    big = (1 << 40) + 5
    h = flat([inv_r(0, [3, 7]), rd(0, {3: (big, 2), 7: None}), {"type": "info", "process": "nemesis", "f": "kill"}])
    assert h.n_events == 2
    pl = h.payload[h.payload_off[1]:h.payload_off[1] + h.payload_len[1]].reshape(-1, 3)
    assert pl[:, 0].tolist() == [H.counter_key(3, 0), H.counter_key(3, 1)] == [6, 7]
    vals = (pl[:, 2].astype(np.int64) << 32) | (pl[:, 1].astype(np.int64) & 0xFFFFFFFF)
    assert vals.tolist() == [big, 2]
    assert h.payload_len[0] == -1   # the invocation carries no value


def test_flatten_negative_counter_round_trips():
    h = flat([inv_r(0, [1]), rd(0, {1: (-3, -(1 << 62))})])
    pl = h.payload.reshape(-1, 3)
    vals = (pl[:, 2].astype(np.int64) << 32) | (pl[:, 1].astype(np.int64) & 0xFFFFFFFF)
    assert vals.tolist() == [-3, -(1 << 62)]


def test_flatten_drops_lookup_transfers_and_non_ok_read_values():
    ops = [{"type": "invoke", "process": 0, "f": "txn", "value": [["l-t", 1, None]]},
           {"type": "ok", "process": 0, "f": "txn", "value": [["l-t", 1, {}]]},
           inv_r(1, [1]), rd(1, {1: (1, 1)}, typ="info")]
    h = flat(ops)
    assert h.n_events == 2 and h.payload_len.tolist() == [-1, -1]


@pytest.mark.parametrize("bad", [
    [rd(0, {-1: (0, 0)})], [rd(0, {1 << 30: (0, 0)})], [rd(0, {1: (1 << 63, 0)})],
    [{"type": "ok", "process": 0, "f": "read", "value": {1: 2}}],
    [{"type": "ok", "process": 0, "f": "txn", "value": [["x", 1, None]]}],
])
def test_flatten_rejects_malformed_input(bad):
    with pytest.raises(ValueError):
        flat(bad)


# ---- synthetic ledger-counter histories -----------------------------------------------------------------------
@pytest.mark.parametrize("stale", [False, True])
def test_ledger_counter_form_matches_the_bank_form(stale):
    spec = synth.SynthSpec("bank", 600, 8, 3, p_info=0.05, stale_read=stale)
    b, c = synth.generate(spec), synth.generate_ledger_counters(spec)
    for name in ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "shard_off", "key_ids"):
        assert np.array_equal(getattr(b, name), getattr(c, name)), name
    assert c.meta["mutated_op_index"] == b.meta["mutated_op_index"]
    reads = np.nonzero((b.type == H.T_OK) & (b.f == H.F_READ))[0]
    assert len(reads) > 100
    for e in reads:
        bal = b.payload[b.payload_off[e]:b.payload_off[e] + b.payload_len[e]].reshape(-1, 2)
        tri = c.payload[c.payload_off[e]:c.payload_off[e] + c.payload_len[e]].reshape(-1, 2, 3)
        assert np.array_equal(tri[:, 0, 0] // 2, bal[:, 0])
        assert np.array_equal(tri[:, 1, 1] - tri[:, 0, 1], bal[:, 1])


def test_synthetic_variants_against_the_oracle():
    spec = synth.SynthSpec("bank", 1500, 16, 2, tau_think_ns=10e6)
    assert M.check_monotonic_keys(synth.generate_ledger_counters(spec))["valid"] == H.VALID
    h = synth.generate_ledger_counters(spec, fractured=True)
    assert h.meta["fractured_op_index"] >= 0
    g, p = both(h)
    assert g["shards"] == p["shards"]


# ---- ABI ------------------------------------------------------------------------------------------------------
def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(9) == ctypes.sizeof(abi.CMonoShard) == 72
    assert lib.jtb_struct_size(10) == ctypes.sizeof(abi.CMonoResult) == 32
