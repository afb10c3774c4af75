"""An independent verifier of the serial-witness check's proofs: plain numpy over the flattened history (the
ledger-lookups form) and commit_read, never the library or the oracle.  For every VALID shard it

  - recomputes the monotonic-key order of the :ok reads (sum of the values, then invocation, stable over completion
    order);
  - replays every read's counters from the transfers commit_read puts at or before it in that order;
  - runs the greedy real-time pass (P_j = max(P_{j-1}, iv(r_j), iv(t) for the transfers first seen by r_j); each read
    needs P_j < cp(r_j), each transfer first seen by r_j with j >= 2 P_{j-1} < cp(t), each transfer after the last read
    P_n < cp(t); cp = infinity for an op that did not complete :ok);
  - checks that no :fail transfer commits, that every :ok one does, and that a transfer committed "freely" moves no
    counter a read observes.

Every transfer of a shard that is not VALID must be SW_NEVER.  Everything is vectorised, so a 10^6-op history takes
about a second."""
from __future__ import annotations

import numpy as np

from jepsen_tigerbeetle_b200 import abi
from jepsen_tigerbeetle_b200 import history as H

NO_CP = np.iinfo(np.int64).max


def _shard(h, s: int):
    """The shard's transfers (history order) and :ok reads (completion order) as numpy arrays."""
    lo, hi = int(h.shard_off[s]), int(h.shard_off[s + 1])
    typ, f = h.type[lo:hi].astype(np.int64), h.f[lo:hi].astype(np.int64)
    proc, plen = h.process[lo:hi].astype(np.int64), h.payload_len[lo:hi].astype(np.int64)
    poff, idx = h.payload_off[lo:hi].astype(np.int64), h.index[lo:hi].astype(np.int64)
    n = hi - lo
    pos = np.arange(n)
    # each event's previous and next event of the same process
    order = np.lexsort((pos, proc))
    same = proc[order][1:] == proc[order][:-1]
    nxt, prv = np.full(n, -1), np.full(n, -1)
    nxt[order[:-1][same]] = order[1:][same]
    prv[order[1:][same]] = order[:-1][same]
    # transfers: the records of the transfer invokes
    ti = np.nonzero((typ == H.T_INVOKE) & (f == H.F_TRANSFER) & (proc >= 0) & (plen > 0))[0]
    nrec = plen[ti] // 5
    ev = np.repeat(ti, nrec)
    first = np.repeat(poff[ti], nrec) + 5 * (np.arange(int(nrec.sum())) - np.repeat(np.cumsum(nrec) - nrec, nrec))
    rec = h.payload[first[:, None] + np.arange(5)].astype(np.int64) if len(first) else np.zeros((0, 5), np.int64)
    comp = nxt[ev]
    fate = np.where((comp >= 0) & (typ[np.maximum(comp, 0)] != H.T_INVOKE), typ[np.maximum(comp, 0)], -1)
    T = {"inv": ev, "fate": fate, "cp": np.where(fate == H.T_OK, comp, NO_CP), "debit": rec[:, 2], "credit": rec[:, 3],
         "amount": rec[:, 4], "id": (rec[:, 1] << 32) | (rec[:, 0] & 0xffffffff)}
    # :ok reads and their (key, value) triples
    ri = np.nonzero((typ == H.T_OK) & (f == H.F_READ) & (proc >= 0) & (plen >= 0))[0]
    p = prv[ri]
    inv = np.where((p >= 0) & (typ[np.maximum(p, 0)] == H.T_INVOKE), p, -1)
    ntrip = plen[ri] // 3
    rrow = np.repeat(np.arange(len(ri)), ntrip)
    tfirst = np.repeat(poff[ri], ntrip) + 3 * (np.arange(int(ntrip.sum())) - np.repeat(np.cumsum(ntrip) - ntrip, ntrip))
    key = h.payload[tfirst].astype(np.int64)
    val = (h.payload[tfirst + 1].astype(np.int64) & 0xffffffff) | (h.payload[tfirst + 2].astype(np.int64) << 32)
    R = {"inv": inv, "cp": ri, "cidx": idx[ri], "row": rrow, "key": key, "val": val, "ntrip": ntrip}
    return T, R


def verify(h, result: dict) -> None:
    """Assert that commit_read in `result` (a check_serial_witness dict with witness=True) proves every VALID shard."""
    cr = np.asarray(result["commit_read"], np.int64)
    at = 0
    for s, sh in enumerate(result["shards"]):
        T, R = _shard(h, s)
        nT = len(T["inv"])
        c = cr[at:at + nT]
        at += nT
        if sh["valid"] != H.VALID:
            assert np.all(c == abi.SW_NEVER), (s, "a shard that is not VALID commits a transfer")
            continue
        _verify_shard(s, T, R, c)
    assert at == len(cr), "commit_read has an entry per transfer micro-op"


def _verify_shard(s: int, T: dict, R: dict, c: np.ndarray) -> None:
    fate = T["fate"]
    committed = c >= 0
    assert not np.any((fate == H.T_FAIL) & (c != abi.SW_NEVER)), (s, "a :fail transfer commits")
    assert not np.any((fate == H.T_OK) & (c == abi.SW_NEVER)), (s, "an :ok transfer never commits")
    assert not np.any((fate != H.T_OK) & ((c == abi.SW_AFTER) | (c == abi.SW_FREE))), (s, "a crashed transfer after or free")
    n = len(R["cp"])
    keys = np.unique(R["key"])
    K = len(keys)
    if n:
        assert np.all(R["ntrip"] == K), (s, "a partial read in a VALID shard")
    jd = np.searchsorted(keys, 2 * T["debit"]) if K else np.zeros(len(fate), np.int64)
    jc = np.searchsorted(keys, 2 * T["credit"] + 1) if K else np.zeros(len(fate), np.int64)
    od = (jd < K) & (keys[np.minimum(jd, K - 1)] == 2 * T["debit"]) if K else np.zeros(len(fate), bool)
    oc = (jc < K) & (keys[np.minimum(jc, K - 1)] == 2 * T["credit"] + 1) if K else np.zeros(len(fate), bool)
    moves = (T["amount"] > 0) & (od | oc)
    assert not np.any((c == abi.SW_FREE) & moves), (s, "a transfer committed freely moves an observed counter")
    if n == 0:
        assert not np.any(committed | (c == abi.SW_AFTER)), (s, "a transfer commits in a shard without reads")
        return
    # the read matrix and the order
    V = np.zeros((n, K), np.int64)
    V[R["row"], np.searchsorted(keys, R["key"])] = R["val"]
    assert not K or np.abs(V).max() < 1 << 54, (s, "counters too large for int64 sums")
    ordr = np.lexsort((R["inv"], V.sum(axis=1)))   # stable: completion order among equal (sum, invocation)
    rank = np.empty(n, np.int64)
    rank[ordr] = np.arange(n)
    # each committed transfer's read: by completion :index
    by_idx = {int(x): r for r, x in enumerate(R["cidx"])}
    tr = np.array([rank[by_idx[int(x)]] if x >= 0 else -1 for x in c.tolist()], np.int64)
    assert np.all((tr >= 0) == committed), (s, "commit_read names something that is not an :ok read")
    # replay
    D = np.zeros((n, K), np.int64)
    m = committed & od
    np.add.at(D, (tr[m], jd[m]), T["amount"][m])
    m = committed & oc
    np.add.at(D, (tr[m], jc[m]), T["amount"][m])
    assert np.array_equal(np.cumsum(D, axis=0), V[ordr]), (s, "a read's counters are not the prefix of its commits")
    # real time
    giv = np.full(n, -1, np.int64)
    np.maximum.at(giv, tr[committed], T["inv"][committed])
    gcp = np.full(n, NO_CP, np.int64)
    np.minimum.at(gcp, tr[committed], T["cp"][committed])
    P = np.maximum.accumulate(np.maximum(R["inv"][ordr], giv))
    assert np.all(P < R["cp"][ordr]), (s, "a read's point is not inside its interval")
    assert np.all(P[:-1] < gcp[1:]), (s, "a transfer's point is not inside its interval")
    after = c == abi.SW_AFTER
    assert np.all(P[-1] < T["cp"][after]), (s, "a transfer after the last read completed before it")
