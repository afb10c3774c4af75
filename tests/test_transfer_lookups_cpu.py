"""The transfer-lookup check without a GPU: hand KATs for every kind against both CPU deciders, their soundness against a
brute-force search for a serial explanation, the two deciders against each other, the ledger-lookups flattener (op maps
and EDN), the synthetic lookups histories, the checker maps and the ABI images of the new structs."""
import ctypes
import hashlib

import numpy as np
import pytest

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, checker, edn, synth
from jepsen_tigerbeetle_b200 import history as H
from test_monotonic_cpu import inv_r, rd

FIELDS = ("valid", "n_failures", "n_lookups", "n_records", "n_transfers", "n_reads", "n_violations", "shards")


def _tv(d, c, amount):
    return {"debit-acct": d, "credit-acct": c, "amount": amount}


def tr(p, typ, d, c, amount, tid):
    """A one-transfer [:t ...] txn of process p with id tid."""
    return {"type": typ, "process": p, "f": "txn", "value": [["t", tid, _tv(d, c, amount)]]}


def inv_l(p):
    return {"type": "invoke", "process": p, "f": "txn", "value": [["l-t", None, None]]}


def lk(p, recs, typ="ok"):
    """A lookup completion; recs = [(id, debit, credit, amount)]."""
    return {"type": typ, "process": p, "f": "txn", "value": [["l-t", i, _tv(d, c, a)] for (i, d, c, a) in recs]}


def final(op):
    return dict(op, **{"final?": True})


def ops_idx(ops):
    return [dict(o, index=i) for i, o in enumerate(ops)]


def flat(ops, model="ledger-lookups"):
    return H.flatten_ops(ops_idx(ops), model)


def both(h):
    """TL_LITERAL and TL_SWEEP, which must agree field by field; returns the first."""
    lit = M.check_transfer_lookups(h, M.TL_LITERAL)
    sw = M.check_transfer_lookups(h, M.TL_SWEEP)
    assert {k: lit[k] for k in FIELDS} == {k: sw[k] for k in FIELDS}, (lit, sw)
    return lit


def shard(ops):
    return both(flat(ops))["shards"][0]


def witness(s):
    return (s["witness_index"], s["kind"], s["transfer_id"], s["key"], s["related_index"], s["value"], s["bound"])


def counts(s):
    return {abi.TL_KIND_NAME[k + 1]: n for k, n in enumerate(s["count_by_kind"]) if n}


T1 = [tr(0, "invoke", 1, 2, 1, 1), tr(0, "ok", 1, 2, 1, 1)]   # transfer 1: account 1 -> 2, amount 1, :ok
R1 = (1, 1, 2, 1)                                              # its record
SEEN = {1: (1, 0), 2: (0, 1)}
UNSEEN = {1: (0, 0), 2: (0, 0)}


# ---- KATs, one per kind ---------------------------------------------------------------------------------------------
def test_valid_lookup():
    s = shard(T1 + [inv_l(1), lk(1, [R1])])
    assert (s["valid"], s["n_lookups"], s["n_records"], s["n_transfers"]) == (H.VALID, 1, 1, 1)
    assert witness(s) == (-1, 0, 0, -1, -1, 0, 0)


def test_phantom():
    s = shard(T1 + [inv_l(1), lk(1, [R1, (9, 1, 2, 1), (7, 1, 2, 1)])])
    assert witness(s) == (3, abi.TL_PHANTOM, 7, -1, -1, 0, 0) and counts(s) == {"phantom": 2}


def test_mismatch():
    s = shard(T1 + [inv_l(1), lk(1, [(1, 1, 2, 5)])])
    assert witness(s) == (3, abi.TL_MISMATCH, 1, -1, 0, 0, 0) and counts(s) == {"mismatch": 1}


def test_failed_visible():
    s = shard([tr(0, "invoke", 1, 2, 1, 1), tr(0, "fail", 1, 2, 1, 1), inv_l(1), lk(1, [R1])])
    assert witness(s) == (3, abi.TL_FAILED_VISIBLE, 1, -1, 0, 0, 0) and counts(s) == {"failed-visible": 1}


def test_future():
    s = shard([inv_l(1), lk(1, [R1])] + T1)
    assert witness(s) == (1, abi.TL_FUTURE, 1, -1, 2, 0, 0) and counts(s) == {"future": 1}


def test_duplicate():
    s = shard(T1 + [inv_l(1), lk(1, [R1, R1, R1])])
    assert witness(s) == (3, abi.TL_DUPLICATE, 1, -1, -1, 0, 0) and counts(s) == {"duplicate": 2}


def test_lost():
    s = shard(T1 + [inv_l(1), lk(1, [])])
    assert witness(s) == (3, abi.TL_LOST, 1, -1, 1, 0, 0) and counts(s) == {"lost": 1}
    assert (s["n_lookups"], s["n_records"]) == (1, 0)


def test_vanished():
    """An :info transfer seen by one lookup and gone from a later one."""
    s = shard([tr(0, "invoke", 1, 2, 1, 1), tr(0, "info", 1, 2, 1, 1), inv_l(1), lk(1, [R1]), inv_l(2), lk(2, [])])
    assert witness(s) == (5, abi.TL_VANISHED, 1, -1, 3, 0, 0) and counts(s) == {"vanished": 1}


def test_read_below_lookup():
    s = shard([tr(0, "invoke", 1, 2, 1, 1), tr(0, "info", 1, 2, 1, 1), inv_l(1), lk(1, [R1]), inv_r(2, [1, 2]),
               rd(2, UNSEEN)])
    assert witness(s) == (5, abi.TL_READ_BELOW_LOOKUP, 0, H.counter_key(1, 0), 3, 0, 1)
    assert counts(s) == {"read-below-lookup": 2}


def test_read_above_lookup():
    s = shard([tr(0, "invoke", 1, 2, 1, 1), tr(0, "info", 1, 2, 1, 1), inv_r(2, [1, 2]), rd(2, SEEN), inv_l(1),
               lk(1, [])])
    assert witness(s) == (3, abi.TL_READ_ABOVE_LOOKUP, 0, H.counter_key(1, 0), 5, 1, 0)
    assert counts(s) == {"read-above-lookup": 2}


def test_smallest_code_of_the_earliest_op_wins():
    # the lookup has a phantom, a mismatch and a loss; an earlier read is fine, a later lookup is worse
    ops = T1 + [tr(0, "invoke", 2, 1, 2, 2), tr(0, "ok", 2, 1, 2, 2), inv_l(1),
                lk(1, [(1, 1, 2, 3), (5, 1, 2, 1)]), inv_l(1), lk(1, [])]
    s = shard(ops)
    assert witness(s)[:3] == (5, abi.TL_PHANTOM, 5)
    assert counts(s) == {"phantom": 1, "mismatch": 1, "lost": 1 + 2}


def test_empty_ok_lookup_and_lookup_without_invocation():
    s = shard([inv_l(1), lk(1, [])])
    assert (s["valid"], s["n_lookups"], s["n_records"]) == (H.VALID, 1, 0)
    # a completion without an invoke requires nothing
    assert shard(T1 + [tr(0, "invoke", 2, 1, 1, 2), tr(0, "ok", 2, 1, 1, 2), lk(1, [R1])])["valid"] == H.VALID


def test_multi_transfer_txn():
    two = [["t", 1, _tv(1, 2, 1)], ["t", 2, _tv(2, 1, 3)]]
    ops = [{"type": "invoke", "process": 0, "f": "txn", "value": two},
           {"type": "ok", "process": 0, "f": "txn", "value": two}, inv_l(1)]
    h = flat(ops + [lk(1, [R1, (2, 2, 1, 3)])])
    assert h.payload_len[0] == 10 and (h.a[0], h.b[0], h.c[0]) == (1, 1, 2)
    s = both(h)["shards"][0]
    assert (s["valid"], s["n_transfers"]) == (H.VALID, 2)
    s = shard(ops + [lk(1, [R1])])
    assert witness(s) == (3, abi.TL_LOST, 2, -1, 1, 0, 0)


def test_uncommitted_info_transfer_is_valid_here_but_not_for_the_reference_checker():
    ops = [tr(0, "invoke", 1, 2, 1, 1), tr(0, "info", 1, 2, 1, 1), tr(1, "invoke", 2, 1, 1, 2), tr(1, "ok", 2, 1, 1, 2),
           final(inv_l(1)), final(lk(1, [(2, 2, 1, 1)]))]
    assert shard(ops)["valid"] == H.VALID
    r = checker.lookup_all_invoked_transfers().check({}, ops_idx(ops))
    assert r["valid?"] is False and len(r["suspect-final-lookups"]) == 1


def test_k8_masked_loss_is_lost_here():
    """An :ok transfer lost and a committed :info one on the same key: the final read holds one amount, which K8's
    bounds [1, 2] allow; the final lookup shows which one is missing."""
    ops = T1 + [tr(0, "invoke", 1, 2, 1, 2), tr(0, "info", 1, 2, 1, 2), final(inv_r(1, [1, 2])), final(rd(1, SEEN)),
                final(inv_l(1)), final(lk(1, [(2, 1, 2, 1)]))]
    assert M.check_counter_bounds(flat(ops, "ledger-counters"))["valid"] == H.VALID
    assert M.check_counter_bounds(flat(ops))["valid"] == H.VALID
    s = shard(ops)
    assert witness(s) == (7, abi.TL_LOST, 1, -1, 1, 0, 0) and counts(s) == {"lost": 1}


def test_errors():
    def raises(ops, match, mutate=None):
        h = flat(ops)
        if mutate:
            mutate(h)
        with pytest.raises(RuntimeError, match=match):
            M.check_transfer_lookups(h)

    raises([tr(0, "invoke", 1, 2, -1, 1)], "negative amount")
    raises([tr(0, "invoke", 1, 1 << 30, 1, 1)], "outside")
    raises([tr(0, "invoke", 1, 2, 1, 1), tr(1, "invoke", 1, 2, 1, 1)], "two transfer invokes")
    raises([tr(0, "invoke", 1, 2, 1, 1)], "without ids", lambda h: h.payload_len.__setitem__(0, -1))
    raises([tr(0, "invoke", 1, 2, 1, 1)], "multiple of 5", lambda h: h.payload_len.__setitem__(0, 4))
    raises(T1 + [inv_l(1), lk(1, [R1])], "multiple of 5", lambda h: h.payload_len.__setitem__(3, 3))
    raises([inv_r(0, [1]), rd(0, {1: (1, 0)})], "payload", lambda h: h.payload_len.__setitem__(1, 5))
    with pytest.raises(RuntimeError, match="reserved"):
        M.check_transfer_lookups(flat(T1), flags=1)


# ---- flattening ---------------------------------------------------------------------------------------------------
def test_flattening_keeps_the_counter_form_and_adds_records():
    ops = T1 + [inv_l(1), lk(1, [R1]), inv_r(2, [1, 2]), rd(2, SEEN), {"type": "invoke", "process": 0, "f": "txn",
                                                                        "value": [["t", (1 << 40) + 3, _tv(2, 1, 4)]]}]
    h, c = flat(ops), flat([o for o in ops if o["value"][0][0] != "l-t"], "ledger-counters")
    assert h.f.tolist() == [H.F_TRANSFER, H.F_TRANSFER, H.F_LOOKUP, H.F_LOOKUP, H.F_READ, H.F_READ, H.F_TRANSFER]
    assert h.payload_len.tolist() == [5, -1, -1, 5, -1, 12, 5]
    assert h.payload[:10].tolist() == [1, 0, 1, 2, 1, 1, 0, 1, 2, 1]
    assert H.transfer_id(*h.payload[22:24]) == (1 << 40) + 3
    keep = h.f != H.F_LOOKUP
    for name in ("type", "f", "process", "a", "b", "c"):
        assert np.array_equal(getattr(h, name)[keep], getattr(c, name)), name
    assert h.meta["multi_transfer_txns"] == 0


def test_edn_history_with_lookups():
    text = """
{:type :invoke, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 1}]], :process 0, :index 0}
{:type :ok, :f :txn, :value [[:t 1 {:debit-acct 1, :credit-acct 2, :amount 1}]], :process 0, :index 1}
{:type :invoke, :f :txn, :value [[:l-t nil nil]], :process 1, :index 2, :final? true}
{:type :ok, :f :txn, :value [[:l-t 1 {:debit-acct 1, :credit-acct 2, :amount 1}]], :process 1, :index 3, :final? true}
{:type :invoke, :f :txn, :value [[:l-t nil nil]], :process 1, :index 4, :final? true}
{:type :ok, :f :txn, :value [], :process 1, :index 5, :final? true}
"""
    ops = edn.read_history(text)
    h = H.flatten_ops(ops, "ledger-lookups")
    assert h.f.tolist() == [H.F_TRANSFER, H.F_TRANSFER] + [H.F_LOOKUP] * 4
    assert h.flags.tolist() == [0, 0, 1, 1, 1, 1] and h.payload_len.tolist() == [5, -1, -1, 5, -1, 0]
    s = both(h)["shards"][0]
    assert witness(s) == (5, abi.TL_LOST, 1, -1, 1, 0, 0)


# ---- soundness: a serial explanation means VALID ----------------------------------------------------------------
def random_tiny(rng):
    """A random tiny history (<= 2 accounts, <= 6 ops) of transfers (ids 1, 2, ...), reads and lookups with :ok, :info,
    :fail and never-completed transfers.  Transfers take effect at their completion (an :info one half the time);
    reads and lookups return what took effect before their completion; most histories get one mutation.
    Returns (op maps, op records for the brute force)."""
    n_acct, n_proc, n_ops = int(rng.integers(1, 3)), int(rng.integers(1, 4)), int(rng.integers(1, 7))
    ops, recs, open_ops, started, applied = [], [], {}, 0, []
    while started < n_ops or (open_ops and rng.random() < 0.7):
        p = int(rng.integers(0, n_proc))
        if p in open_ops:
            r = open_ops.pop(p)
            r["comp"] = len(ops)
            if r["kind"] == "t":
                r["fate"] = str(rng.choice(["ok", "ok", "info", "fail"]))
                if r["fate"] == "ok" or (r["fate"] == "info" and rng.random() < 0.5):
                    applied.append(r)
                ops.append(tr(p, r["fate"], r["b"], r["c"], r["a"], r["id"]))
            elif r["kind"] == "r":
                r["fate"] = "ok"
                d = [sum(t["a"] for t in applied if t["b"] == a + 1) for a in range(n_acct)]
                c = [sum(t["a"] for t in applied if t["c"] == a + 1) for a in range(n_acct)]
                r["values"] = {H.counter_key(a + 1, 0): d[a] for a in range(n_acct)}
                r["values"].update({H.counter_key(a + 1, 1): c[a] for a in range(n_acct)})
                ops.append(rd(p, {a + 1: (d[a], c[a]) for a in range(n_acct)}))
            else:
                r["fate"] = "ok"
                r["recs"] = [(t["id"], t["b"], t["c"], t["a"]) for t in applied]
                ops.append(lk(p, r["recs"]))
        elif started < n_ops:
            started += 1
            x = rng.random()
            if x < 0.3:
                r = {"kind": "r", "inv": len(ops), "comp": None, "fate": None}
                ops.append(inv_r(p, list(range(1, n_acct + 1))))
            elif x < 0.55:
                r = {"kind": "l", "inv": len(ops), "comp": None, "fate": None}
                ops.append(inv_l(p))
            else:
                b, c = int(rng.integers(1, n_acct + 1)), int(rng.integers(1, n_acct + 1))
                r = {"kind": "t", "inv": len(ops), "comp": None, "fate": None, "a": int(rng.integers(0, 3)), "b": b,
                     "c": c, "id": sum(1 for q in recs if q["kind"] == "t") + 1}
                ops.append(tr(p, "invoke", b, c, r["a"], r["id"]))
            open_ops[p] = r
            recs.append(r)
    done = [r for r in recs if r["kind"] in ("l", "r") and r["fate"] == "ok"]
    if done and rng.random() < 0.6:
        r = done[int(rng.integers(0, len(done)))]
        op = ops[r["comp"]]
        if r["kind"] == "r":
            k = int(rng.integers(0, len(op["value"])))
            acct = op["value"][k][2]
            acct["debits-posted"] += int(rng.choice([-1, 1]))
            r["values"][H.counter_key(op["value"][k][1], 0)] = acct["debits-posted"]
        else:
            m = int(rng.integers(0, 4))
            n_t = sum(1 for q in recs if q["kind"] == "t")
            if m == 0 and r["recs"]:
                r["recs"] = r["recs"][1:]
            elif m == 1 and r["recs"]:
                r["recs"] = r["recs"] + r["recs"][:1]
            elif m == 2 and n_t:
                pick = int(rng.integers(1, n_t + 1))
                t = next(q for q in recs if q["kind"] == "t" and q["id"] == pick)
                r["recs"] = r["recs"] + [(t["id"], t["b"], t["c"], t["a"])]
            elif r["recs"]:
                i, d, c, a = r["recs"][0]
                r["recs"] = [(i, d, c, a + 1)] + r["recs"][1:]
            ops[r["comp"]] = lk(op["process"], r["recs"])
    return ops, recs


def explainable(recs) -> bool:
    """Is there a serial order of points inside the op intervals that explains every :ok read and :ok lookup?  Each
    committed transfer has an id-enqueue point and, after it, a commit point (:ok transfers commit, :fail ones do not,
    :info and never-completed ones may); each :ok read and lookup has one point.  A read returns the counters of the
    transfers committed before it; a lookup returns, once each and as issued, exactly the transfers committed before it
    (every committed transfer's id was enqueued before its commit)."""
    must = [r for r in recs if r["fate"] == "ok"]
    maybe = [r for r in recs if r["kind"] == "t" and r["fate"] in ("info", None)]
    for pick in range(1 << len(maybe)):
        ops = must + [m for i, m in enumerate(maybe) if pick >> i & 1]
        pts = []   # (op, is_enqueue)
        for o in ops:
            if o["kind"] == "t":
                pts.append((o, True))
            pts.append((o, False))
        n = len(pts)
        last = {id(o): j for j, (o, _) in enumerate(pts)}   # an op is done when its last point is
        pred = []
        for j, (x, enq) in enumerate(pts):
            m = 0
            for y in ops:
                if y["comp"] is not None and y["comp"] < x["inv"]:
                    m |= 1 << last[id(y)]
            if x["kind"] == "t" and not enq:
                m |= 1 << (j - 1)
            pred.append(m)
        reach = {0}
        for mask in range(1 << n):
            if mask not in reach:
                continue
            done_t = [o for j, (o, enq) in enumerate(pts) if mask >> j & 1 and o["kind"] == "t" and not enq]
            for j, (x, enq) in enumerate(pts):
                if mask >> j & 1 or pred[j] & ~mask:
                    continue
                if x["kind"] == "r" and not enq:
                    cnt: dict[int, int] = {}
                    for t in done_t:
                        cnt[H.counter_key(t["b"], 0)] = cnt.get(H.counter_key(t["b"], 0), 0) + t["a"]
                        cnt[H.counter_key(t["c"], 1)] = cnt.get(H.counter_key(t["c"], 1), 0) + t["a"]
                    if any(cnt.get(k, 0) != v for k, v in x["values"].items()):
                        continue
                if x["kind"] == "l" and sorted(x["recs"]) != sorted((t["id"], t["b"], t["c"], t["a"]) for t in done_t):
                    continue
                reach.add(mask | 1 << j)
        if (1 << n) - 1 in reach:
            return True
    return False


def test_sound_against_brute_force():
    rng = np.random.default_rng(29)
    verdicts = {H.VALID: 0, H.INVALID: 0}
    kinds = set()
    explained = 0
    for _ in range(2000):
        ops, recs = random_tiny(rng)
        s = both(flat(ops))["shards"][0]
        verdicts[s["valid"]] += 1
        kinds.add(s["kind"])
        if explainable(recs):
            explained += 1
            assert s["valid"] == H.VALID, ops
    assert verdicts[H.VALID] > 200 and verdicts[H.INVALID] > 200, verdicts
    assert explained > 200
    assert kinds >= {0, abi.TL_MISMATCH, abi.TL_DUPLICATE, abi.TL_LOST, abi.TL_FAILED_VISIBLE,
                     abi.TL_READ_BELOW_LOOKUP, abi.TL_READ_ABOVE_LOOKUP}, kinds


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


@pytest.mark.parametrize("make,spec,kw,digest", [
    (synth.generate, synth.SynthSpec("bank", 2000, 16, 3, p_info=0.05), {},
     "aa1a754bdd4349f83a63a8b92d2cd00da9e3c85a837aca6bdc11569be89424de"),
    (synth.generate_ledger_counters, synth.SynthSpec("bank", 3000, 16, 5, p_info=0.05, stale_read=True), {},
     "f5ccd4f7b64a016cc1d4e8d0f3fe6e3d370913fc3395861e062f01ccb1ee8ca7"),
    (synth.generate_ledger_counters, synth.SynthSpec("bank", 1500, 16, 3, final_reads=True), {"lost_transfer": True},
     "f82cf2682ee8cc89d13a4f829353c6a27bf1b7c7940dd51609bb08d95371a4bd"),
])
def test_default_outputs_are_unchanged(make, spec, kw, digest):
    """Digests of generate() and generate_ledger_counters() output taken before the lookups form existed."""
    assert _digest(make(spec, **kw)) == digest


def test_lookups_history_extends_the_counter_history():
    spec = synth.SynthSpec("bank", 1500, 8, 2, p_info=0.05, final_reads=True)
    c = synth.generate_ledger_counters(spec)
    h = synth.generate_ledger_lookups(spec)
    n = c.n_events
    for name in ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c"):
        assert np.array_equal(getattr(h, name)[:n], getattr(c, name)), name
    tin = np.nonzero((c.f == H.F_TRANSFER) & (c.type == H.T_INVOKE))[0]
    assert np.array_equal(h.payload_len[tin], np.full(len(tin), 5))
    recs = np.stack([h.payload[h.payload_off[e]:h.payload_off[e] + 5] for e in tin])
    assert recs[:, 0].tolist() == list(range(1, len(tin) + 1))
    assert np.array_equal(recs[:, 2:], np.stack([c.b[tin], c.c[tin], c.a[tin]], 1))
    tail = slice(n, h.n_events)
    assert h.n_events - n == 2 * 8 and np.all(h.f[tail] == H.F_LOOKUP) and np.all(h.flags[tail] == H.FLAG_FINAL)
    r = both(h)
    assert r["valid"] == H.VALID and r["n_lookups"] == 8


# mutation -> (the kind it adds, the witness kind).  A vanished record also leaves the last lookup's sums below the
# final read, which completes earlier and so is the witness.
MUTATIONS = {"lost_transfer": (abi.TL_LOST,) * 2, "phantom_record": (abi.TL_PHANTOM,) * 2,
             "mismatched_record": (abi.TL_MISMATCH,) * 2, "vanished_record": (abi.TL_VANISHED, abi.TL_READ_ABOVE_LOOKUP),
             "inflated_read": (abi.TL_READ_ABOVE_LOOKUP,) * 2}


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_mutations(mutation):
    spec = synth.SynthSpec("bank", 1500, 8, 3, p_info=0.05, final_reads=True)
    base = synth.generate_ledger_lookups(spec)
    h = synth.generate_ledger_lookups(spec, **{mutation: True})
    for name in ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c"):
        assert np.array_equal(getattr(h, name), getattr(base, name)), name
    r = both(h)
    kind, wkind = MUTATIONS[mutation]
    s = r["shards"][0]
    assert r["valid"] == H.INVALID and s["kind"] == wkind and s["count_by_kind"][kind - 1] > 0, r
    assert counts(both(base)["shards"][0]) == {}


def test_mid_history_lookups():
    spec = synth.SynthSpec("bank", 300, 6, 4, p_info=0.05, final_reads=True)
    h = synth.generate_ledger_lookups(spec, p_lookup=0.05)
    r = both(h)
    assert r["valid"] == H.VALID and r["n_lookups"] > 6 + 5
    h = synth.generate_ledger_lookups(spec, p_lookup=0.05, lost_transfer=True)
    assert both(h)["valid"] == H.INVALID


@pytest.mark.parametrize("seed", [1, 2])
def test_oracles_agree_on_c3_size(seed):
    for kw in ({}, {"lost_transfer": True}, {"inflated_read": True}):
        h = synth.generate_ledger_lookups(synth.SynthSpec("bank", 10000, 32, seed, p_info=0.02, final_reads=True), **kw)
        r = both(h)
        assert r["n_lookups"] == 32 and r["valid"] == (H.INVALID if kw else H.VALID)


# ---- checker maps -------------------------------------------------------------------------------------------------
class _FakeCtx:
    """A context that answers with the CPU oracle, so the result maps can be checked without a GPU."""

    def check_transfer_lookups(self, h):
        return M.check_transfer_lookups(h)


def test_checker_result_map():
    ops = ops_idx(T1 + [inv_l(1), lk(1, [])])
    r = checker.transfer_lookup_checker(ctx=_FakeCtx()).check({}, ops)
    assert r["valid?"] is False
    assert (r["lookup-count"], r["record-count"], r["transfer-count"], r["read-count"], r["error-count"]) == (
        1, 0, 1, 0, 1)
    assert r["errors"] == {"lost": 1}
    assert r["op"] == {"index": 3}
    assert r["error"] == {"type": "lost", "transfer-id": 1, "related": {"index": 1}}
    ops = ops_idx([tr(0, "invoke", 1, 2, 1, 1), tr(0, "info", 1, 2, 1, 1), inv_r(2, [1, 2]), rd(2, SEEN), inv_l(1),
                   lk(1, [])])
    r = checker.transfer_lookup_checker(ctx=_FakeCtx()).check({}, ops)
    assert r["error"] == {"type": "read-above-lookup", "key": [1, "debits-posted"], "value": 1, "bound": 0,
                          "related": {"index": 5}}
    ok = ops_idx(T1 + [inv_l(1), lk(1, [R1])])
    r = checker.transfer_lookup_checker(ctx=_FakeCtx()).check({}, ok)
    assert r["valid?"] is True and r["errors"] == {} and "op" not in r and "error" not in r
    comp = checker.ledger_checker(ctx=_FakeCtx(), linear=False, transfer_lookups=True)
    assert "transfer-lookups" in comp.checkers
    assert "transfer-lookups" not in checker.ledger_checker(linear=False).checkers
    ind = checker.independent_checker(checker.transfer_lookup_checker(ctx=_FakeCtx()))
    assert ind._model() == "ledger-lookups"


# ---- ABI ------------------------------------------------------------------------------------------------------
def test_struct_sizes_against_the_library():
    from jepsen_tigerbeetle_b200 import native
    lib = native.lib()
    assert lib.jtb_struct_size(13) == ctypes.sizeof(abi.CTlShard) == 136
    assert lib.jtb_struct_size(14) == ctypes.sizeof(abi.CTlResult) == 64


def test_jni_shim_reports_errors_without_a_device():
    """jtb.Native.checkTransferLookups through the JNI shim and a fake JNIEnv: a null context throws."""
    fj = _tl_fakejvm()
    with pytest.raises(fj.JavaException):
        fj._result(fj.lib().fj_check_transfer_lookups(0, fj.jhistory(flat(T1))), np.int64)


def _tl_fakejvm():
    """tests/fakejvm.py pointed at fake_jvm_tl.c (the driver of checkTransferLookups)."""
    import ctypes as C
    import importlib.util
    import os

    import fakejvm
    here = os.path.dirname(os.path.abspath(fakejvm.__file__))
    spec = importlib.util.spec_from_file_location("fakejvm_tl", fakejvm.__file__)
    fj = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fj)
    fj._SO = os.path.join(here, "native", "libjtb_fakejvm_tl.so")
    fj._SRCS = [os.path.join(here, "native", "fake_jvm_tl.c")] + fj._SRCS[1:]
    fj._DEPS = fj._DEPS + [os.path.join(here, "native", "fake_jvm_tl.c"), os.path.join(here, "native", "fake_jvm.c")]
    L = fj.lib()
    L.fj_check_transfer_lookups.restype = C.c_void_p
    L.fj_check_transfer_lookups.argtypes = [C.c_longlong, C.c_void_p]
    return fj
