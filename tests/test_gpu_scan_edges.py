"""set-full, bank totals and the key partition on the device at their kernels' boundaries (scan_shapes.py), compared
with the CPU oracle (set-full, bank) and numpy (partition) field by field."""
import ctypes as C

import numpy as np
import pytest

import scan_shapes as S
from jepsen_tigerbeetle_b200 import abi, native
from jepsen_tigerbeetle_b200 import history as H
from jepsen_tigerbeetle_b200.native import NativeError

pytestmark = pytest.mark.gpu


def sf_equal(g, o):
    assert g["valid"] == o["valid"]
    for s, (gs, os_) in enumerate(zip(g["shards"], o["shards"])):
        assert gs == os_, s
    assert len(g["shards"]) == len(o["shards"]) and g["n_failures"] == o["n_failures"]
    assert g["raia_valid"] == o["raia_valid"] and g["suspect_final_reads"] == o["suspect_final_reads"]
    for k in ("elem_off", "elem_id", "elem_outcome", "elem_latency_ms", "elem_dup_count"):
        assert np.array_equal(g[k], o[k]), k


def bank_equal(g, o):
    for k in g:
        if not k.startswith("seconds"):
            assert g[k] == o[k], k


def bank_model(neg_ok=True, accounts=S.ACCOUNTS):
    return H.make_model(H.MODEL_BANK, accounts=accounts, negative_balances_ok=neg_ok)


@pytest.fixture(scope="module")
def many_keys():
    return S.sf_many_keys()


# ---- set-full -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(S.SF_SHAPES))
def test_set_full_shapes(gpu_ctx, oracle_mod, name):
    h = S.SF_SHAPES[name]()
    for lin in (True, False):
        sf_equal(gpu_ctx.check_set_full(h, lin), oracle_mod.check_set_full(h, lin))


def test_set_full_add_free_duplicate(gpu_ctx):
    """0:inv read, 0:ok read [7 7] with no :add anywhere: the repeat is :duplicated and the key :invalid."""
    g = gpu_ctx.check_set_full(S.sf_add_free_duplicate())
    assert g["shards"][0]["duplicated_count"] == 1
    assert g["valid"] == H.INVALID


def test_set_full_hand_answers(gpu_ctx):
    g = gpu_ctx.check_set_full(S.sf_latency())
    assert g["elem_latency_ms"].tolist() == [0, 1, 1]
    assert [s["valid"] for s in g["shards"]] == [H.VALID, H.INVALID, H.INVALID]
    g = gpu_ctx.check_set_full(S.sf_finals())
    assert [x["missing"] for x in g["suspect_final_reads"]] == [[968, 969], [0], [9]]
    g = gpu_ctx.check_set_full(S.sf_duplicates())
    assert [s["duplicated_count"] for s in g["shards"]] == [4, 1, 1, 1, 0]


def test_set_full_more_shards_than_a_grid_dimension(gpu_ctx, oracle_mod, many_keys):
    """70,000 keys: the column scan covers more shards than gridDim.z can hold in one launch."""
    h = many_keys
    for lin in (True, False):
        g = gpu_ctx.check_set_full(h, lin)
        sf_equal(g, oracle_mod.check_set_full(h, lin))
    k = np.arange(h.n_shards)
    assert sum(s["lost_count"] for s in g["shards"]) == int((k % 7 == 3).sum())
    assert g["shards"][-1]["lost_count"] == int((h.n_shards - 1) % 7 == 3)


def test_set_full_buffer_reuse_with_stale_contents(gpu_ctx, oracle_mod, many_keys):
    """The context's cached device buffers hold the previous call's contents: big, empty and small histories in turn."""
    seq = [S.sf_reads(1025, 4097, seed=1), S.Script().flat(), S.sf_add_free_duplicate(), many_keys, S.sf_elements(33),
           S.sf_id_tables(), S.sf_degenerate(), S.sf_reads(1025, 4097, seed=1), S.sf_finals()]
    expect = [oracle_mod.check_set_full(h) for h in seq]
    for h, o in zip(seq, expect):
        sf_equal(gpu_ctx.check_set_full(h), o)


# ---- bank totals ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(S.BANK_SHAPES))
def test_bank_shapes(gpu_ctx, oracle_mod, name):
    build, total = S.BANK_SHAPES[name]
    h = build()
    for m in (bank_model(True), bank_model(False), bank_model(accounts=())):
        bank_equal(gpu_ctx.check_bank_totals(h, m, total), oracle_mod.check_bank_totals(h, m, total))


def test_bank_hand_answers(gpu_ctx):
    g = gpu_ctx.check_bank_totals(S.bank_float_tie(), bank_model(), S.FLOAT_TIE_TOTAL)
    assert g["worst_index_by_type"][3] == 1 and (g["lowest_index"], g["highest_index"]) == (1, 3)
    g = gpu_ctx.check_bank_totals(S.bank_precedence(), bank_model(False), 0)
    assert g["worst_index_by_type"] == [-1, 1, 3, 5, 7] and (g["lowest_index"], g["highest_index"]) == (5, 5)
    g = gpu_ctx.check_bank_totals(S.bank_extremes(), bank_model(False), 3)
    assert (g["lowest_total"], g["highest_total"]) == (8 * (S.INT32_MIN + 1), 8 * S.INT32_MAX)


def test_bank_rejects_account_counts_outside_the_model(gpu_ctx, oracle_mod):
    h = S.bank_outcomes()
    for n in (-1, H.MAX_ACCOUNTS + 1):
        m = bank_model()
        m.n_accounts = n
        ch, res = H.as_c_history(h), abi.CBankResult()
        assert native.lib().jtb_check_bank_totals(gpu_ctx._h, C.addressof(ch), C.addressof(m), C.c_int64(0),
                                                  C.addressof(res)) < 0
        assert "0..8 accounts" in gpu_ctx._err()
        bank_equal(gpu_ctx.check_bank_totals(h, bank_model(), 0), oracle_mod.check_bank_totals(h, bank_model(), 0))


# ---- partition and ledger balances ----------------------------------------------------------------------------------
@pytest.mark.parametrize("n", S.PARTITION_SIZES)
@pytest.mark.parametrize("kind", ["specials", "equal", "distinct"])
def test_partition_shapes(gpu_ctx, n, kind):
    keys = S.partition_keys(n, kind)
    r = gpu_ctx.partition_by_key(keys)
    order = np.argsort(keys, kind="stable").astype(np.int32)
    assert np.array_equal(r["order"], order)
    ids, first = np.unique(keys[order], return_index=True)
    assert np.array_equal(r["key_ids"], ids)
    assert np.array_equal(r["shard_off"], np.concatenate([first, [n]]).astype(np.int64))


def _partition(ctx, keys, cap):
    n = keys.shape[0]
    order = np.empty(n, np.int32)
    off = np.full(cap + 1, -7, np.int64)
    ids = np.full(max(cap, 1), -7, np.int64)
    nk = C.c_int32(-1)
    rc = native.lib().jtb_partition_by_key(ctx._h, C.c_int64(n), keys.ctypes.data_as(C.c_void_p),
                                           order.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p),
                                           ids.ctypes.data_as(C.c_void_p), C.c_int32(cap), C.byref(nk))
    return rc, order, off, ids, nk.value


def test_partition_key_cap(gpu_ctx, oracle_mod):
    """key_cap exactly the number of keys succeeds; one less fails with "key_cap too small" and leaves the context
    usable."""
    keys = S.partition_keys(257, "specials")
    n_keys = len(np.unique(keys))
    rc, order, off, ids, nk = _partition(gpu_ctx, keys, n_keys)
    assert rc == 0 and nk == n_keys
    assert np.array_equal(ids[:nk], np.unique(keys)) and off[nk] == keys.shape[0]
    rc, _, _, _, nk = _partition(gpu_ctx, keys, n_keys - 1)
    assert rc < 0 and nk == 0 and "key_cap too small" in gpu_ctx._err()
    r = gpu_ctx.partition_by_key(keys)
    assert np.array_equal(r["key_ids"], np.unique(keys))
    h = S.sf_duplicates()
    sf_equal(gpu_ctx.check_set_full(h), oracle_mod.check_set_full(h))


def test_ledger_balances_truncate_to_int32(gpu_ctx):
    c, d, expect = S.wide_balances()
    assert np.array_equal(gpu_ctx.ledger_balances(c, d), expect)
    for n in S.PARTITION_SIZES:
        rng = np.random.default_rng(n)
        c = rng.integers(-(2 ** 40), 2 ** 40, n)
        d = rng.integers(-(2 ** 40), 2 ** 40, n)
        assert np.array_equal(gpu_ctx.ledger_balances(c, d), (c - d).astype(np.int32))
