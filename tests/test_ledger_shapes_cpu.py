"""The full-width transforms and cap shapes of tests/ledger_shapes.py without a GPU: every builder and transform makes a
well-formed history that reaches the value or count it is named for and changes nothing else; the CPU oracles give the
hand-derived answers at the caps of K7-K13; and the oracles (and the brute references, on the small shapes) return the
mapped result on every transformed history."""
import numpy as np
import pytest

import ledger_shapes as L
import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi, synth
from jepsen_tigerbeetle_b200 import history as H
from test_transfer_lookups_cpu import tr

EVENT_FIELDS = ("type", "f", "flags", "process", "index", "time_ns", "payload_off", "payload_len", "shard_off",
                "key_ids")
BRUTE = {"mono": {"algo": M.MONO_PAIRS}, "cb": {"algo": M.CB_LITERAL}, "tl": {"algo": M.TL_LITERAL},
         "rx": {"algo": M.RX_BRUTE}, "rg": {"algo": M.RG_BRUTE}}


def families():
    """Small histories of both ledger forms, with crashed transfers, mid-history lookups and several shards."""
    spec = synth.SynthSpec("bank", 600, 8, 2, p_info=0.05, final_reads=True)
    yield "counters", synth.generate_ledger_counters(spec)
    yield "counters stale", synth.generate_ledger_counters(synth.SynthSpec("bank", 600, 8, 3, stale_read=True))
    yield "lookups", synth.generate_ledger_lookups(spec, p_lookup=0.05)
    yield "lookups torn", synth.generate_ledger_lookups(spec, torn_pair=True)
    yield "64 accounts", synth.generate_ledger_lookups(synth.SynthSpec("bank", 800, 16, 4, n_accounts=64,
                                                                       p_info=0.02, final_reads=True))
    yield "shards", H.concat_keys([synth.generate_ledger_lookups(synth.SynthSpec(
        "bank", 300, 8, s, tau_think_ns=5e6, p_info=0.05, final_reads=True), split_amount=s == 2) for s in (1, 2, 3)])


def checks_of(h):
    return L.CHECKS if h.meta["model"] == "ledger-lookups" else ("mono", "cb")


def unchanged_except(h, g, payload_at=(), fields=()):
    for f in EVENT_FIELDS + tuple(x for x in ("a", "b", "c") if x not in fields):
        assert np.array_equal(getattr(h, f), getattr(g, f)), f
    keep = np.ones(len(h.payload), bool)
    keep[np.asarray(payload_at, np.int64)] = False
    assert np.array_equal(h.payload[keep], g.payload[keep])


# ---- the transforms ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,h", list(families()), ids=[n for n, _ in families()])
def test_transforms_are_well_formed(name, h):
    tri, rec = L.read_triples(h), L.transfer_records(h)
    t = L.is_transfer(h)
    g, _ = L.scale(h)
    g.validate()
    c = L.scale_factor(h)
    assert lands_near_int32_max(g) and c * L.max_amount(h) <= L.INT32_MAX
    unchanged_except(h, g, np.concatenate([rec + 4, tri + 1, tri + 2]), ("a",))
    assert np.array_equal(g.a[t], h.a[t] * c) and np.array_equal(g.payload[rec + 4], h.payload[rec + 4] * c)
    assert np.array_equal(L._get64(g.payload, tri), L._get64(h.payload, tri) * c)
    assert np.abs(L._get64(g.payload, tri)).max() < 1 << 54
    g, _ = L.remap_ids(h)
    g.validate()
    unchanged_except(h, g, np.concatenate([rec, rec + 1]))
    ids = [H.transfer_id(lo, hi) for lo, hi in zip(g.payload[rec], g.payload[rec + 1])]
    assert ids == [L.ID_MAP(H.transfer_id(lo, hi)) for lo, hi in zip(h.payload[rec], h.payload[rec + 1])]
    if len(rec):
        assert min(ids) < 0 and (g.payload[rec] < 0).any() and (g.payload[rec] >= 0).any()
    g, _ = L.shift_accounts(h)
    g.validate()
    unchanged_except(h, g, np.concatenate([rec + 2, rec + 3, tri]), ("b", "c"))
    assert L.max_account(g) == L.TOP_ACCOUNT
    d = L.TOP_ACCOUNT - L.max_account(h)
    assert np.array_equal(g.b[t], h.b[t] + d) and np.array_equal(g.payload[tri], h.payload[tri] + 2 * d)
    g, _ = L.offset_counters(h)
    g.validate()
    unchanged_except(h, g, np.concatenate([tri + 1, tri + 2]))
    diff = L._get64(g.payload, tri) - L._get64(h.payload, tri)
    assert set(np.unique(np.abs(diff)).tolist()) == {L.BIG}


def lands_near_int32_max(g):
    """The largest amount lands within a few units of INT32_MAX."""
    return L.INT32_MAX - L.max_amount(g) < 8


def test_full_width_flattening():
    """What the transforms put in the payload is what the flattener makes of the same op maps."""
    h = L.units(3, 3)
    g, _ = L.shift_accounts(L.remap_ids(L.scale(h)[0])[0])
    c, d = L.scale_factor(h), L.TOP_ACCOUNT - 2
    ops = [tr(p, "invoke", 1 + d, 2 + d, c, L.ID_MAP(p + 1)) for p in range(3)]
    ops += [L.inv_r(3, [1 + d, 2 + d]), L.rd(3, {1 + d: (3 * c, 0), 2 + d: (0, 3 * c)})]
    ops += [tr(p, "ok", 1 + d, 2 + d, c, L.ID_MAP(p + 1)) for p in range(3)]
    want = L.flat(ops)
    for f in EVENT_FIELDS + ("a", "b", "c", "payload"):
        assert np.array_equal(getattr(g, f), getattr(want, f)), f
    assert int(g.payload[L.read_triples(g)].max()) == L.INT32_MAX


@pytest.mark.parametrize("name,h", list(families()), ids=[n for n, _ in families()])
def test_oracles_are_invariant(name, h):
    for check in checks_of(h):
        base = L.oracle(check, h)
        for tname, fn in L.TRANSFORMS.items():
            g, expect = fn(h)
            assert L.comparable(L.oracle(check, g)) == L.comparable(expect(check, base)), (check, tname)
    g, expect = L.offset_counters(h)
    assert L.comparable(L.oracle("mono", g)) == L.comparable(expect("mono", L.oracle("mono", h)))
    if h.n_shards == 1 and M.check_monotonic_keys(h)["shards"][0]["cause"] == 0:   # full-key reads
        g, expect = L.offset_counters(h, L.wrap_offsets(h))
        assert L.comparable(L.oracle("mono", g)) == L.comparable(expect("mono", L.oracle("mono", h)))
        assert sum(L.wrap_offsets(h).values()) < 0


SMALL = {"int32 max": L.int32_max_amounts(0), "int32 max + 1": L.int32_max_amounts(1), "zero": L.zero_amount(),
         "branching": L.branching(), "keys 33": L.keys_per_read(33), "placement chain": L.placement_chain(3),
         "witness chain": L.witness_chain(3)}


@pytest.mark.parametrize("name", list(SMALL))
def test_brute_references_are_invariant(name):
    h = SMALL[name]
    for check, kw in BRUTE.items():
        base = L.oracle(check, h, **kw)
        for tname, fn in L.TRANSFORMS.items():
            g, expect = fn(h)
            assert L.comparable(L.oracle(check, g, **kw)) == L.comparable(expect(check, base)), (check, tname)
    base = M.check_transfer_placement(h, M.TP_BRUTE)
    for fn in L.TRANSFORMS.values():
        g, _ = fn(h)
        b = M.check_transfer_placement(g, M.TP_BRUTE)
        assert (b["valid"], b["n_reads"], b["n_transfers"]) == (base["valid"], base["n_reads"], base["n_transfers"])


# ---- the caps, by hand ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nt", [1, 31, 32, 33, 64, 65, 255, 256, 257])
def test_keys_per_read(nt):
    h = L.keys_per_read(nt)
    h.validate()
    tri = L.read_triples(h)
    assert len(tri) == 2 * nt and len(np.unique(h.payload[tri])) == nt
    for check in ("mono", "cb", "tl"):
        assert L.oracle(check, h)["valid"] == H.VALID, check
    want = (H.UNKNOWN, 1) if nt > abi.RX_MAX_KEYS else (H.VALID, 0)
    rx = L.oracle("rx", h)
    assert (rx["valid"], rx["n_undecided"]) == (H.UNKNOWN, 2) if nt > abi.RX_MAX_KEYS else (H.VALID, 0)
    for check in ("rg", "tp"):
        r = L.oracle(check, h)
        assert (r["valid"], min(r["n_undecided"], 1)) == want, check
    assert L.oracle("sw", h)["shards"][0]["cause"] == (abi.CAUSE_UNDECIDED if nt > abi.RX_MAX_KEYS else 0)


@pytest.mark.parametrize("n", [127, 128, 129])
@pytest.mark.parametrize("n_ok", [63, 64, 65, 95, 96, 97])
def test_gather_cap(n, n_ok):
    h = L.units(n, n, n_ok)
    assert np.count_nonzero((h.type == H.T_INFO) & L.is_transfer(h)) == n - n_ok
    for check in ("rx", "rg", "tp"):
        r = L.oracle(check, h)
        if n > abi.RX_MAX_GATHER:
            assert (r["valid"], r["n_undecided"], r["nodes"]) == (H.UNKNOWN, 1, 0), check
        else:
            assert (r["valid"], r["n_explained"], r["shards"][0]["nodes"] > 0) == (H.VALID, 1, True), check
    assert L.oracle("sw", L.units(n, n, n_ok))["valid"] == (H.UNKNOWN if n > abi.RX_MAX_GATHER else H.VALID)


def test_amount_zero_is_not_gathered():
    """A transfer of amount 0 beside 128 gathered ones neither counts toward the cap nor becomes a free candidate."""
    assert L.oracle("rx", L.units(128, 128, 64, zeros=1))["n_explained"] == 1
    assert L.oracle("rx", L.units(64, 20, zeros=1))["n_explained"] == 1
    r = L.oracle("sw", L.zero_amount())
    assert r["valid"] == H.VALID and r["commit_read"].tolist() == [5, abi.SW_FREE, 5, abi.SW_NEVER]


@pytest.mark.parametrize("nf", [63, 64, 65])
def test_free_cap(nf):
    h = L.units(nf, 20)
    for check in ("rx", "rg", "tp"):
        r = L.oracle(check, h)
        if nf > abi.RX_MAX_FREE:
            assert (r["valid"], r["n_undecided"]) == (H.UNKNOWN, 1), check
        else:
            assert (r["valid"], r["n_explained"], r["shards"][0]["nodes"] % 21) == (H.VALID, 1, 0), check


def test_node_budget():
    h = L.branching()
    n = L.oracle("rx", h)["nodes"]
    assert n == L.oracle("rg", h)["nodes"] == 13
    for check in ("rx", "rg"):
        assert L.oracle(check, h, max_nodes=n - 1)["n_undecided"] == 1
        for mx in (n, n + 1):
            assert L.oracle(check, h, max_nodes=mx)["n_explained"] == 1
    assert L.oracle("tp", h, max_nodes=n - 1)["valid"] == H.UNKNOWN
    assert L.oracle("sw", h, max_nodes=n)["valid"] == H.VALID


def test_max_rounds():
    h = L.placement_chain(5)
    r = L.oracle("tp", h)
    assert (r["valid"], r["rounds"], r["n_placed"]) == (H.VALID, 6, 5)
    assert L.oracle("tp", h, max_rounds=5)["n_placed"] == 5
    assert L.oracle("tp", h, max_rounds=4)["n_placed"] == 4
    h = L.witness_chain(5)
    r = L.oracle("sw", h)
    assert (r["valid"], r["rounds"]) == (H.VALID, 5)
    assert L.oracle("sw", h, max_rounds=6)["valid"] == H.VALID
    assert L.oracle("sw", h, max_rounds=4)["shards"][0]["cause"] == abi.CAUSE_NO_WITNESS


def test_witness_choice_follows_the_signed_id_order():
    """With ids on both sides of zero the first solution of every gap is the transfer of the smallest signed id."""
    h = L.witness_chain(5)
    base = L.oracle("sw", h)
    g, expect = L.remap_ids(h, (1 << 29) - 3)
    ids = [H.transfer_id(lo, hi) for lo, hi in zip(g.payload[L.transfer_records(g)], g.payload[L.transfer_records(g) + 1])]
    assert min(ids) < 0 < max(ids)
    assert L.comparable(L.oracle("sw", g)) == L.comparable(expect("sw", base))


def test_int32_max_amounts():
    r = L.oracle("rx", L.int32_max_amounts(0))
    assert (r["valid"], r["n_explained"]) == (H.VALID, 1)
    s = L.oracle("rx", L.int32_max_amounts(1))["shards"][0]
    assert (s["kind"], s["key"], s["value"], s["must_sum"]) == (abi.RX_KEY, 2, 2 ** 32 - 1, 0)
    s = L.oracle("rg", L.int32_max_amounts(1))["shards"][0]
    assert (s["kind"], s["key"], s["delta"]) == (abi.RG_KEY, 2, 2 ** 32 - 1)


def test_many_shards():
    h = L.many_shards(70_000)
    assert h.n_shards == 70_000
    assert np.count_nonzero(np.diff(h.shard_off) == 2) > 60_000   # one read, no transfer
    for check in ("rx", "rg", "tp"):
        r = L.oracle(check, h)
        bad = [s for s, q in enumerate(r["shards"]) if q["valid"] != H.VALID]
        assert bad == [s for s in range(70_000) if s % 1001 == 500], check
