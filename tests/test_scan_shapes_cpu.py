"""The boundary-shape builders of scan_shapes.py and the CPU oracle's answers on them (no device).

The GPU comparison in test_gpu_scan_edges.py trusts the oracle; here the oracle itself is held to answers derived by
hand on the small shapes, and every builder to a well-formed history."""
import numpy as np
import pytest

import scan_shapes as S
from jepsen_tigerbeetle_b200 import history as H

OUTCOME_NEVER_READ, OUTCOME_STABLE, OUTCOME_LOST = 0, 1, 2   # JTB_SF_*


def well_formed(h: H.FlatHistory):
    """CSR layout, one :index per event of a shard, and every completion closing an open invoke of its process with
    the same :f (a process has at most one op open)."""
    h.validate()
    assert h.key_ids.shape == (h.n_shards,)
    for s in range(h.n_shards):
        lo, hi = int(h.shard_off[s]), int(h.shard_off[s + 1])
        assert len(set(h.index[lo:hi].tolist())) == hi - lo
        assert np.all(np.diff(h.index[lo:hi]) > 0)
        open_ = {}
        for e in range(lo, hi):
            p = int(h.process[e])
            if p < 0:
                continue
            if h.type[e] == H.T_INVOKE:
                assert p not in open_, (s, e)
                open_[p] = int(h.f[e])
            else:
                assert open_.pop(p, None) == int(h.f[e]), (s, e)
            if h.payload_len[e] >= 0:
                assert h.payload_off[e] + h.payload_len[e] <= h.payload.shape[0]


@pytest.mark.parametrize("name", list(S.SF_SHAPES))
def test_set_full_shapes_are_well_formed(name):
    well_formed(S.SF_SHAPES[name]())


@pytest.mark.parametrize("name", list(S.BANK_SHAPES))
def test_bank_shapes_are_well_formed(name):
    h = S.BANK_SHAPES[name][0]()
    well_formed(h)
    assert h.meta["model"] == "bank"


def test_set_full_shapes_reach_their_edges():
    """The shapes hold what their names promise: element counts, read counts, chunk-crossing reads, the n_elig values."""
    for n in S.ELEMENT_COUNTS:
        assert S.tracked_ids(S.sf_elements(n), 0) == list(range(2 * n, 3 * n))
    for r in S.READ_COUNTS + (1025,):
        h = S.sf_reads(r, 4097 if r == 1025 else 70)
        pending, inv_by_completion = {}, []
        for e in range(h.n_events):
            if h.f[e] == H.F_READ:
                if h.type[e] == H.T_INVOKE:
                    pending[int(h.process[e])] = int(h.index[e])
                else:
                    inv_by_completion.append(pending.pop(int(h.process[e])))
        assert len(inv_by_completion) == r
        assert not np.all(np.diff(inv_by_completion) > 0)     # completion order is not invocation order
    h = S.sf_elig()
    add_inv = np.sort(h.index[(h.f == H.F_ADD) & (h.type == H.T_INVOKE)])
    ok_idx = h.index[(h.f == H.F_READ) & (h.type == H.T_OK)]
    n_elig = set(np.searchsorted(add_inv, ok_idx).tolist())
    assert set(S.ELIG_TARGETS) <= n_elig
    h = S.sf_many_keys()
    assert h.n_shards == 70_000 > S.GRID_YZ_MAX


def test_id_table_paths():
    """The span rule of run_set_full's id table (direct iff span <= 4n + 1024) and the path each id-table shard takes."""
    assert S.lookup_path(list(range(7)) + [4 * 8 + 1023]) == "direct"
    assert S.lookup_path(list(range(7)) + [4 * 8 + 1024]) == "sorted"
    assert S.lookup_path([S.INT32_MIN, S.INT32_MAX]) == "sorted"
    assert S.lookup_path([]) == "none"
    h = S.sf_id_tables()
    paths = [S.lookup_path(S.tracked_ids(h, s)) for s in range(h.n_shards)]
    assert paths == h.meta["lookup"] == ["direct", "sorted", "direct", "sorted", "sorted"]
    assert S.INT32_MIN in S.tracked_ids(h, 4) and S.INT32_MAX in S.tracked_ids(h, 4)
    assert min(S.tracked_ids(h, 2)) < 0


def test_oracle_add_free_duplicate(oracle_mod):
    """0:inv read, 0:ok read [7 7]: (frequencies v) sees 7 twice -> duplicated-count 1, :valid? false."""
    for lin in (True, False):
        o = oracle_mod.check_set_full(S.sf_add_free_duplicate(), lin)
        sh = o["shards"][0]
        assert (sh["attempt_count"], sh["duplicated_count"], sh["valid"]) == (0, 1, H.INVALID)
        assert o["valid"] == H.INVALID and len(o["elem_id"]) == 0


def test_oracle_duplicates(oracle_mod):
    o = oracle_mod.check_set_full(S.sf_duplicates())
    assert [s["duplicated_count"] for s in o["shards"]] == [4, 1, 1, 1, 0]
    assert [s["valid"] for s in o["shards"]] == [H.INVALID] * 4 + [H.UNKNOWN]
    off = o["elem_off"]
    dup0 = dict(zip(o["elem_id"][off[0]:off[1]].tolist(), o["elem_dup_count"][off[0]:off[1]].tolist()))
    assert {k: v for k, v in dup0.items() if v} == {0: 2, 31: 3, 32: 2, 63: 4}
    # an id repeated before its add was invoked still counts for that element
    assert o["elem_id"][off[2]:off[3]].tolist() == [5] and o["elem_dup_count"][off[2]:off[3]].tolist() == [2]


def test_oracle_latency_boundary(oracle_mod):
    """stable_time - known_time of 999,999, 1,000,000 and 1,000,001 ns: latencies 0, 1, 1 ms."""
    h = S.sf_latency()
    o = oracle_mod.check_set_full(h, True)
    assert o["elem_outcome"].tolist() == [OUTCOME_STABLE] * 3
    assert o["elem_latency_ms"].tolist() == [0, 1, 1]
    assert [s["stale_count"] for s in o["shards"]] == [0, 1, 1]
    assert [s["stable_latency_max_ms"] for s in o["shards"]] == [0, 1, 1]
    assert [s["valid"] for s in o["shards"]] == [H.VALID, H.INVALID, H.INVALID]
    assert [s["valid"] for s in oracle_mod.check_set_full(h, False)["shards"]] == [H.VALID] * 3


def test_oracle_finals(oracle_mod):
    o = oracle_mod.check_set_full(S.sf_finals())
    assert o["raia_valid"] == H.INVALID
    assert [s["suspect_final_reads"] for s in o["shards"]] == [1, 0, 2]
    assert [sorted(x["missing"]) for x in o["suspect_final_reads"]] == [[968, 969], [0], [9]]


def test_oracle_degenerate_and_many_keys(oracle_mod):
    o = oracle_mod.check_set_full(S.sf_degenerate())
    assert [s["attempt_count"] for s in o["shards"]] == [0, 0, 3, 0, 2]
    assert [s["valid"] for s in o["shards"]] == [H.UNKNOWN, H.UNKNOWN, H.UNKNOWN, H.UNKNOWN, H.INVALID]
    h = S.sf_many_keys()
    o = oracle_mod.check_set_full(h)
    k = np.arange(70_000)
    lost, dup = k % 7 == 3, (k % 11 == 5) & (k % 7 != 3)
    assert sum(s["lost_count"] for s in o["shards"]) == int(lost.sum())
    assert sum(s["duplicated_count"] for s in o["shards"]) == int(dup.sum())
    assert o["n_failures"] == int((lost | dup).sum())


def _bank_oracle(oracle_mod, h, total, neg_ok=True, accounts=S.ACCOUNTS):
    return oracle_mod.check_bank_totals(h, H.make_model(H.MODEL_BANK, accounts=accounts,
                                                        negative_balances_ok=neg_ok), total)


def test_oracle_bank_outcomes(oracle_mod):
    h = S.bank_outcomes()
    o = _bank_oracle(oracle_mod, h, 0, neg_ok=False)
    assert o["count_by_type"] == [0, 1, 1, 1, 1]
    assert o["first_index_by_type"] == [-1, 3, 5, 7, 9] and o["error_count"] == 4
    o = _bank_oracle(oracle_mod, h, 0, neg_ok=True)
    assert o["count_by_type"] == [0, 1, 1, 1, 0]
    o = _bank_oracle(oracle_mod, h, 0, accounts=())
    assert o["count_by_type"] == [0, 5, 0, 0, 0] and o["first_error_index"] == 1


def test_oracle_bank_precedence_and_ties(oracle_mod):
    """unexpected-key > nil-balance > wrong-total > negative-value; equal badness and equal totals go to the earliest
    :index (read k has :index 2k + 1)."""
    o = _bank_oracle(oracle_mod, S.bank_precedence(), 0, neg_ok=False)
    types = S.BANK_PRECEDENCE_TYPES
    assert o["count_by_type"] == [0] + [types.count(t) for t in (1, 2, 3, 4)]
    first = [2 * types.index(t) + 1 for t in (1, 2, 3, 4)]
    last = [2 * (len(types) - 1 - types[::-1].index(t)) + 1 for t in (1, 2, 3, 4)]
    assert o["first_index_by_type"] == [-1] + first and o["last_index_by_type"] == [-1] + last
    assert o["worst_index_by_type"] == [-1, 1, 3, 5, 7]
    assert (o["lowest_total"], o["highest_total"], o["lowest_index"], o["highest_index"]) == (7, 7, 5, 5)
    assert (o["first_error_index"], o["first_error_type"]) == (1, 1)
    assert o["reference_throws"] == 1 and o["valid"] == H.UNKNOWN


def test_oracle_bank_float_tie(oracle_mod):
    """Ratios that differ as doubles but not after (float ...): the earlier read is the worst."""
    d1, d2 = S.FLOAT_TIE_DIFFS
    T = S.FLOAT_TIE_TOTAL
    assert d1 / T != d2 / T and np.float32(d1 / T) == np.float32(d2 / T)
    o = _bank_oracle(oracle_mod, S.bank_float_tie(), T)
    assert o["count_by_type"][3] == 2 and o["worst_index_by_type"][3] == 1
    assert (o["lowest_index"], o["highest_index"]) == (1, 3)
    assert o["valid"] == H.INVALID and o["reference_throws"] == 0


def test_oracle_bank_extremes(oracle_mod):
    o = _bank_oracle(oracle_mod, S.bank_extremes(), 3, neg_ok=False)
    assert o["read_count"] == 8
    assert o["lowest_total"] == 8 * (S.INT32_MIN + 1) and o["highest_total"] == 8 * S.INT32_MAX
    assert o["count_by_type"] == [0, 0, 1, 7, 0]       # every read without a nil sums to something other than 3
    assert o["last_index_by_type"][3] == 2 * 2 + 2 * 7 + 1   # the all-zero read after the two transfers
    o = _bank_oracle(oracle_mod, S.bank_no_reads(), 0)
    assert (o["read_count"], o["error_count"], o["valid"]) == (0, 0, H.VALID)


def test_partition_shapes():
    for n in S.PARTITION_SIZES:
        for kind in ("specials", "equal", "distinct"):
            k = S.partition_keys(n, kind)
            assert k.dtype == np.int64 and k.shape == (n,)
            if kind == "distinct":
                assert len(np.unique(k)) == n
                assert set(S.SPECIAL_KEYS[:min(4, n)].tolist()) <= set(k.tolist())
            if kind == "equal":
                assert len(np.unique(k)) == 1
    assert set(S.SPECIAL_KEYS.tolist()) <= set(S.partition_keys(1000, "specials").tolist())
    c, d, expect = S.wide_balances()
    assert expect.tolist() == [S.INT32_MIN, S.INT32_MAX, 2, 0, S.INT32_MIN, S.INT32_MIN, 0, 3, -2]
    assert np.array_equal(expect, (c - d).astype(np.int32))
