"""The ledger checks K7-K13 on the GPU with full-width values and at their kernels' caps (tests/ledger_shapes.py).

Every shape and every transformed copy of the synthetic families is compared with the CPU oracle field by field (every
field but the timings, commit_read entry by entry), and the device is compared with itself: its result on scale(h),
remap_ids(h) and shift_accounts(h) must be its result on h mapped through the transform, which holds even where the
oracle and the device would share a width bug.  Every K13 VALID is re-checked by tests/serial_witness.py."""
import pytest

import ledger_shapes as L
from jepsen_tigerbeetle_b200 import abi, synth
from jepsen_tigerbeetle_b200 import history as H
from serial_witness import verify

pytestmark = pytest.mark.gpu


def agree(ctx, check, h, **kw):
    g = L.device(ctx, check, h, **kw)
    assert L.comparable(g) == L.comparable(L.oracle(check, h, **kw)), check
    if check == "sw":
        verify(h, g)
    return g


def invariant(ctx, check, h, checks_oracle=True, **kw):
    """The device on h and on every transform of h: against the oracle and against itself."""
    base = agree(ctx, check, h, **kw) if checks_oracle else L.device(ctx, check, h, **kw)
    for name, fn in L.TRANSFORMS.items():
        g, expect = fn(h)
        got = agree(ctx, check, g, **kw) if checks_oracle else L.device(ctx, check, g, **kw)
        if check == "sw":
            verify(g, got)
        assert L.comparable(got) == L.comparable(expect(check, base)), (check, name)
    return base


# ---- the synthetic families, transformed -----------------------------------------------------------------------------
C3 = synth.SynthSpec("bank", 10000, 32, 1, final_reads=True)
LOOKUP_MUTATIONS = ("lost_transfer", "torn_transfer", "torn_pair", "split_amount")


def family(name):
    """(ledger-counters form, ledger-lookups form) of one family."""
    if name == "c3 valid":
        return synth.generate_ledger_counters(C3), synth.generate_ledger_lookups(C3)
    if name == "c3 stale":
        spec = synth.SynthSpec("bank", 10000, 32, 1, final_reads=True, stale_read=True)
        return synth.generate_ledger_counters(spec), synth.generate_ledger_lookups(spec)
    if name == "c3 fractured":
        return synth.generate_ledger_counters(C3, fractured=True), None
    if name.startswith("c3 "):
        m = name[3:]
        return (synth.generate_ledger_counters(C3, lost_transfer=True) if m == "lost_transfer" else None,
                synth.generate_ledger_lookups(C3, **{m: True}))
    if name == "p_info 0.02":
        spec = synth.SynthSpec("bank", 10000, 32, 1, p_info=0.02, final_reads=True)
        return synth.generate_ledger_counters(spec), synth.generate_ledger_lookups(spec)
    if name == "mid-history lookups":
        spec = synth.SynthSpec("bank", 600, 8, 2, p_info=0.05, final_reads=True)
        return None, H.concat_keys([synth.generate_ledger_lookups(spec, p_lookup=0.05, **kw)
                                    for kw in ({}, {"lost_transfer": True}, {"torn_pair": True})])
    if name == "64 accounts":
        spec = synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, p_info=0.02, final_reads=True)
        return synth.generate_ledger_counters(spec), synth.generate_ledger_lookups(spec)
    assert name == "multi-shard"
    muts = {2: "torn_transfer", 5: "split_amount", 6: "torn_pair"}
    specs = [synth.SynthSpec("bank", 1500, 8, s, tau_think_ns=5e6, p_info=0.05, final_reads=True) for s in range(1, 9)]
    return (H.concat_keys([synth.generate_ledger_counters(sp) for sp in specs]),
            H.concat_keys([synth.generate_ledger_lookups(sp, **({muts[s + 1]: True} if s + 1 in muts else {}))
                           for s, sp in enumerate(specs)]))


FAMILIES = ("c3 valid", "c3 stale", "c3 fractured") + tuple("c3 " + m for m in LOOKUP_MUTATIONS) + (
    "p_info 0.02", "mid-history lookups", "64 accounts", "multi-shard")


@pytest.mark.parametrize("name", FAMILIES)
def test_families(gpu_ctx, name):
    counters, lookups = family(name)
    if counters is not None:
        for check in ("mono", "cb"):
            invariant(gpu_ctx, check, counters)
    if lookups is not None:
        for check in L.CHECKS:
            invariant(gpu_ctx, check, lookups)


# ---- K7's 128-bit sums -----------------------------------------------------------------------------------------------
def test_offset_counters(gpu_ctx):
    """Counters of +-(2^62 - 2^50): the read sums and the warp's partial sums leave int64, and the order stays; with
    wrap_offsets the order of half the reads rests on the carry out of the low 64 bits."""
    stale = synth.SynthSpec("bank", 4000, 32, 4, n_accounts=64, final_reads=True, stale_read=True)
    for h in (family("64 accounts")[0], synth.generate_ledger_counters(stale), L.keys_per_read(256),
              L.keys_per_read(257)):
        for per_key in (None, L.wrap_offsets(h)):
            g, expect = L.offset_counters(h, per_key)
            assert L.comparable(agree(gpu_ctx, "mono", g)) == L.comparable(expect("mono", agree(gpu_ctx, "mono", h)))


@pytest.mark.parametrize("stale", [False, True])
def test_offset_counters_million_ops(gpu_ctx, stale):
    h = synth.generate_ledger_counters(synth.SynthSpec("bank", 1_000_000, 32, 1, final_reads=True, stale_read=stale))
    g, expect = L.offset_counters(h)
    base = gpu_ctx.check_monotonic_keys(h)
    assert L.comparable(gpu_ctx.check_monotonic_keys(g)) == L.comparable(expect("mono", base))
    assert (base["valid"] == H.INVALID) == stale


# ---- the caps ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nt", [1, 31, 32, 33, 64, 65, 255, 256, 257])
def test_keys_per_read(gpu_ctx, nt):
    h = L.keys_per_read(nt)
    for check in L.CHECKS:
        invariant(gpu_ctx, check, h)


@pytest.mark.parametrize("n", [127, 128, 129])
def test_gather_cap(gpu_ctx, n):
    for n_ok in (63, 64, 65, 95, 96, 97):
        h = L.units(n, n, n_ok)
        for check in ("rx", "rg", "tp", "sw"):
            r = invariant(gpu_ctx, check, h)
            assert (r["valid"] == H.VALID) == (n <= abi.RX_MAX_GATHER), (check, n_ok)
    h = L.units(n, n, 64, zeros=1)
    assert agree(gpu_ctx, "rx", h)["valid"] == (H.VALID if n <= abi.RX_MAX_GATHER else H.UNKNOWN)


@pytest.mark.parametrize("nf", [63, 64, 65])
def test_free_cap(gpu_ctx, nf):
    for h in (L.units(nf, 20), L.units(nf, 20, zeros=1)):
        for check in ("rx", "rg", "tp", "sw"):
            r = invariant(gpu_ctx, check, h)
            assert (r["valid"] == H.VALID) == (nf <= abi.RX_MAX_FREE), check


def test_node_budget(gpu_ctx):
    h = L.branching()
    n = L.oracle("rx", h)["nodes"]
    for mx in (n - 1, n, n + 1):
        for check in ("rx", "rg", "tp", "sw"):
            r = invariant(gpu_ctx, check, h, max_nodes=mx)
            assert (r["valid"] == H.VALID) == (mx >= n), (check, mx)


def test_max_rounds(gpu_ctx):
    h = L.placement_chain(5)
    R = L.oracle("tp", h)["rounds"]
    for mr in (R - 1, R, R + 1):
        assert invariant(gpu_ctx, "tp", h, max_rounds=mr)["rounds"] == min(mr, R)
    h = L.witness_chain(5)
    R = L.oracle("sw", h)["rounds"]
    for mr in (R - 1, R, R + 1):
        assert (invariant(gpu_ctx, "sw", h, max_rounds=mr)["valid"] == H.VALID) == (mr >= R)
    g, expect = L.remap_ids(h, (1 << 29) - 3)   # ids on both sides of zero: the choice follows the signed order
    assert L.comparable(agree(gpu_ctx, "sw", g)) == L.comparable(expect("sw", agree(gpu_ctx, "sw", h)))


def test_amount_edges(gpu_ctx):
    for extra in (0, 1):
        h = L.int32_max_amounts(extra)
        for check in L.CHECKS:
            invariant(gpu_ctx, check, h)
    s = agree(gpu_ctx, "rx", L.int32_max_amounts(1))["shards"][0]
    assert (s["kind"], s["value"], s["must_sum"]) == (abi.RX_KEY, 2 ** 32 - 1, 0)
    h = L.zero_amount()
    for check in L.CHECKS:
        invariant(gpu_ctx, check, h)
    assert agree(gpu_ctx, "sw", h)["commit_read"].tolist()[1] == abi.SW_FREE


def test_many_shards(gpu_ctx):
    h = L.many_shards(70_000)
    for check in L.CHECKS:
        r = agree(gpu_ctx, check, h)
        assert r["n_failures"] == (0 if check in ("mono", "tl") else 70), check   # the reads that contradict
    for check in ("rx", "rg", "tp"):
        invariant(gpu_ctx, check, h, checks_oracle=False)
