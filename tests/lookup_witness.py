"""An independent verifier of the lookup witness's proofs: plain numpy and Python over the flattened history (the
ledger-lookups form), commit_read and lookup_read, never the library or the oracle.  For every VALID shard it

  - recomputes the monotonic-key order of the :ok reads and replays every read's counters from the transfers
    commit_read puts in the gaps up to it;
  - gives every transfer its gap (a read's position, n after the last read, none) and every :ok lookup the gap
    lookup_read names; a transfer committed "freely" goes after the last read on a shard with lookups;
  - checks each lookup's records (a transfer of the shard with its invocation's debit, credit and amount, no id twice)
    and that it returns every transfer of the earlier gaps, none of the later ones and part of its own;
  - orders each gap: the lookups by how much of the gap they return, which must be nested, each after the transfers it
    is the first to return, then the transfers no lookup returns, then the read; transfers by invocation;
  - runs one greedy real-time pass over that order: P = max(P, iv(op)) < cp(op) for every op.

Every transfer and lookup of a shard that is not VALID must be SW_NEVER."""
from __future__ import annotations

import numpy as np

from jepsen_tigerbeetle_b200 import abi
from jepsen_tigerbeetle_b200 import history as H
from serial_witness import _shard


def _lookups(h, s: int) -> list[dict]:
    """The shard's :ok lookups in completion order: invocation, completion position, :index and records."""
    lo, hi = int(h.shard_off[s]), int(h.shard_off[s + 1])
    last: dict[int, int] = {}
    out = []
    for e in range(lo, hi):
        p = int(h.process[e])
        if p < 0:
            continue
        if h.type[e] == H.T_INVOKE:
            last[p] = e - lo
            continue
        if h.type[e] != H.T_OK or h.f[e] != H.F_LOOKUP or h.payload_len[e] < 0:
            continue
        off, n = int(h.payload_off[e]), int(h.payload_len[e])
        rec = h.payload[off:off + n].astype(np.int64).reshape(-1, 5)
        out.append({"inv": last.get(p, -1), "cp": e - lo, "cidx": int(h.index[e]),
                    "id": (rec[:, 1] << 32) | (rec[:, 0] & 0xffffffff), "rec": rec})
    return out


def verify(h, result: dict) -> None:
    """Assert that commit_read and lookup_read in `result` (a check_lookup_witness dict with witness=True) prove every
    VALID shard."""
    cr = np.asarray(result["commit_read"], np.int64)
    lr = np.asarray(result["lookup_read"], np.int64)
    at = lat = 0
    for s, sh in enumerate(result["shards"]):
        T, R = _shard(h, s)
        L = _lookups(h, s)
        c, lrd = cr[at:at + len(T["inv"])], lr[lat:lat + len(L)]
        at += len(T["inv"])
        lat += len(L)
        if sh["valid"] != H.VALID:
            assert np.all(c == abi.SW_NEVER) and np.all(lrd == abi.SW_NEVER), (s, "a shard that is not VALID commits")
            continue
        _verify_shard(s, T, R, L, c, lrd)
    assert at == len(cr) and lat == len(lr), "one entry per transfer micro-op and per :ok lookup"


def _verify_shard(s, T, R, L, c, lrd) -> None:
    fate = T["fate"]
    nT, n = len(fate), len(R["cp"])
    assert not np.any((fate == H.T_FAIL) & (c != abi.SW_NEVER)), (s, "a :fail transfer commits")
    assert not np.any((fate == H.T_OK) & (c == abi.SW_NEVER)), (s, "an :ok transfer never commits")
    assert not np.any((fate != H.T_OK) & (c == abi.SW_FREE)), (s, "a crashed transfer commits freely")
    keys = np.unique(R["key"])
    K = len(keys)
    if n:
        assert np.all(R["ntrip"] == K), (s, "a partial read in a VALID shard")
    V = np.zeros((n, K), np.int64)
    if n:
        V[R["row"], np.searchsorted(keys, R["key"])] = R["val"]
    ordr = np.lexsort((R["inv"], V.sum(axis=1))) if n else np.zeros(0, np.int64)
    rank = np.empty(n, np.int64)
    rank[ordr] = np.arange(n)
    by_idx = {int(x): int(rank[r]) for r, x in enumerate(R["cidx"])}
    NONE = 1 << 62
    free_at = n if L else NONE
    G = np.array([by_idx[int(x)] if x >= 0 else n if x == abi.SW_AFTER else free_at if x == abi.SW_FREE else NONE
                  for x in c.tolist()], np.int64)
    assert np.all((c < 0) | np.isin(c, R["cidx"])), (s, "commit_read names something that is not an :ok read")
    # the reads' counters
    if n:
        D = np.zeros((n + 1, K), np.int64)
        for acct, side in ((T["debit"], 0), (T["credit"], 1)):
            k = 2 * acct + side
            j = np.searchsorted(keys, k)
            hit = (j < K) & (keys[np.minimum(j, K - 1)] == k) & (G < NONE)
            np.add.at(D, (G[hit], j[hit]), T["amount"][hit])
        assert np.array_equal(np.cumsum(D[:n], axis=0), V[ordr]), (s, "a read's counters are not its commits")
    # the lookups' contents
    tix = {int(i): t for t, i in enumerate(T["id"].tolist())}
    lpos = [by_idx[int(x)] if x >= 0 else n for x in lrd.tolist()]
    assert all(x >= 0 or x == abi.SW_AFTER for x in lrd.tolist()), (s, "lookup_read names no place")
    layer = {}
    gap_lookups: dict[int, list] = {}
    for j, lk in enumerate(L):
        ts = []
        for r, i in zip(lk["rec"], lk["id"].tolist()):
            t = tix.get(int(i))
            assert t is not None, (s, "a lookup record names no transfer")
            assert (T["debit"][t], T["credit"][t], T["amount"][t]) == (r[2], r[3], r[4]), (s, "a mismatched record")
            ts.append(t)
        assert len(set(ts)) == len(ts), (s, "a lookup returns an id twice")
        g = lpos[j]
        shown = np.zeros(nT, bool)
        shown[ts] = True
        assert np.all(shown[G < g]), (s, "a lookup lacks a transfer of an earlier gap")
        assert not np.any(shown & (G > g)), (s, "a lookup returns a transfer of a later gap or one never committed")
        gap_lookups.setdefault(g, []).append((int(np.sum(shown & (G == g))), j, set(np.nonzero(shown & (G == g))[0])))
    # the order inside each gap, and its nesting
    ops = []   # (gap, sub, iv, cp)
    for g, ls in gap_lookups.items():
        ls.sort()
        prev: set = set()
        for r, (a, j, sub) in enumerate(ls):
            assert prev <= sub, (s, "the lookups of one gap are not nested")
            for t in sub - prev:
                layer[t] = r
            prev = sub
            ops.append((g, 2 * r + 1, L[j]["inv"], L[j]["cp"]))
    for t in range(nT):
        if G[t] < NONE:
            ops.append((int(G[t]), 2 * layer[t] if t in layer else 1 << 40, int(T["inv"][t]), int(T["cp"][t])))
    for i in range(n):
        r = int(ordr[i])
        ops.append((i, 1 << 41, int(R["inv"][r]), int(R["cp"][r])))
    ops.sort()
    P = -1 << 62
    for g, sub, iv, cp in ops:
        P = max(P, iv)
        assert P < cp, (s, "an op's point is not inside its interval", g, sub)
