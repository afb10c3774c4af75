"""Full-width value transforms and cap-shaped histories for the ledger checks K7-K13 (plain Python, no device).

Transforms (on the ledger-counters and ledger-lookups forms): each returns (history', expect), where expect(check, r)
maps a result dict r of the original for `check` (one of CHECKS) to the result the transformed history must give.

  scale(h, c)             every amount and every read counter times c: amounts reach INT32_MAX, counters pass 2^40.
                          Every comparison the checks make is homogeneous, so verdicts, witnesses and node counts stay
                          and only the value-like fields (value, bound, must_sum, delta, edge values) scale.
  remap_ids(h)            every transfer id through the increasing ID_MAP: negative ids, ids above 2^32 and low words
                          with the sign bit set.  Only transfer_id fields change.
  shift_accounts(h)       every account up by 2^30 - 1 - max_account, so the top key is INT32_MAX.  Only key fields change.
  offset_counters(h, o)   K7 only, on full-key shards: o[key] added to every read's value of key, so per-read sums and
                          the warp's partial sums leave int64.  Only the edge values change.

Cap shapes (include/jtb_check.h): keys per read, gathered "may" transfers, free candidates after the root pruning, the
node budget, placement and witness rounds, amounts at INT32_MAX and 0, and many shards.
"""
from __future__ import annotations

import numpy as np

import mono_oracle as M
from jepsen_tigerbeetle_b200 import abi
from jepsen_tigerbeetle_b200 import history as H
from test_monotonic_cpu import inv_r, rd
from test_transfer_lookups_cpu import flat, tr
from test_transfer_placement_cpu import script

INT32_MAX = 2 ** 31 - 1
TOP_ACCOUNT = (1 << 30) - 1
CHECKS = ("mono", "cb", "tl", "rx", "rg", "tp", "sw")
BIG = (1 << 62) - (1 << 50)   # offset_counters' magnitude: 2^62 - 2^50


def ID_MAP(i):
    """The increasing id map of remap_ids (numpy int64 arrays or Python ints)."""
    return (i - (1 << 29)) * ((1 << 32) + (1 << 31) + 1)


# ---- payload addressing --------------------------------------------------------------------------------------------
def _starts(h, mask, width):
    """Payload positions of every width-int32 record of the events in mask."""
    ev = np.nonzero(mask & (h.payload_len > 0))[0]
    n = h.payload_len[ev].astype(np.int64) // width
    first = np.repeat(h.payload_off[ev], n)
    inner = np.arange(int(n.sum()), dtype=np.int64) - np.repeat(np.cumsum(n) - n, n)
    return first + width * inner


def read_triples(h):
    """Payload positions of the (key, lo, hi) triples of every :ok read."""
    return _starts(h, (h.type == H.T_OK) & (h.f == H.F_READ), 3)


def transfer_records(h):
    """Payload positions of the (id_lo, id_hi, debit, credit, amount) records of transfer invokes and :ok lookups."""
    mask = ((h.type == H.T_INVOKE) & (h.f == H.F_TRANSFER)) | ((h.type == H.T_OK) & (h.f == H.F_LOOKUP))
    return _starts(h, mask, H.TRANSFER_RECORD)


def _get64(p, at):
    return (p[at + 1].astype(np.int64) & 0xFFFFFFFF) | (p[at + 2].astype(np.int64) << 32)


def _set64(p, at, v):
    v = np.asarray(v, np.int64)
    p[at + 1] = (v & 0xFFFFFFFF).astype(np.uint32).view(np.int32)
    p[at + 2] = (v >> 32).astype(np.int32)


def _copy(h):
    return H.FlatHistory(*(getattr(h, f).copy() for f in ("type", "f", "flags", "process", "index", "time_ns", "a",
                                                           "b", "c", "payload_off", "payload_len", "payload",
                                                           "shard_off", "key_ids")), dict(h.meta))


def is_transfer(h):
    return h.f == H.F_TRANSFER


def max_amount(h):
    rec = transfer_records(h)
    m = int(h.a[is_transfer(h)].max(initial=0))
    return max(m, int(h.payload[rec + 4].max(initial=0)))


def max_account(h):
    t = is_transfer(h)
    rec = transfer_records(h)
    tri = read_triples(h)
    return max(int(h.b[t].max(initial=0)), int(h.c[t].max(initial=0)), int(h.payload[rec + 2].max(initial=0)),
               int(h.payload[rec + 3].max(initial=0)), int((h.payload[tri] // 2).max(initial=0)))


# ---- result mapping ------------------------------------------------------------------------------------------------
def map_result(check, r, value=None, key=None, tid=None):
    """r with the value-like fields through value(), the key fields through key() and the transfer-id fields through
    tid(), each where the check defines it (None: unchanged)."""
    value = value or (lambda v: v)
    key = key or (lambda k: k)
    tid = tid or (lambda i: i)
    out = dict(r)
    out["shards"] = shards = [dict(s) for s in r["shards"]]
    for s in shards:
        if check == "mono":
            s["edges"] = [(k, key(kk), value(v), value(v2)) if k == abi.MONO_EDGE_MONOTONIC else (k, kk, v, v2)
                          for (k, kk, v, v2) in s["edges"]]
        elif check == "cb":
            if s["witness_key"] >= 0:
                s["witness_key"] = key(s["witness_key"])
            s["value"], s["bound"] = value(s["value"]), value(s["bound"])
        elif check == "tl":
            if 1 <= s["kind"] <= 7:
                s["transfer_id"] = tid(s["transfer_id"])
            if s["key"] >= 0:
                s["key"] = key(s["key"])
            s["value"], s["bound"] = value(s["value"]), value(s["bound"])
        elif check == "rx":
            if s["key"] >= 0:
                s["key"] = key(s["key"])
            s["value"], s["must_sum"] = value(s["value"]), value(s["must_sum"])
        elif check in ("rg", "tp"):
            if s["key"] >= 0:
                s["key"] = key(s["key"])
            s["delta"] = value(s["delta"])
            if s["kind"] == abi.RG_DOUBLE or (check == "tp" and s["kind"] == abi.TP_LOST):
                s["transfer_id"] = tid(s["transfer_id"])
        elif check == "sw":
            if s["transfer_id"] != -1:
                s["transfer_id"] = tid(s["transfer_id"])
    return out


# ---- transforms ----------------------------------------------------------------------------------------------------
def scale_factor(h):
    return (2 ** 31 - 1) // max(1, max_amount(h))


def scale(h, c=None):
    c = scale_factor(h) if c is None else c
    g = _copy(h)
    t = is_transfer(g)
    g.a[t] = (g.a[t].astype(np.int64) * c).astype(np.int32)
    rec = transfer_records(g)
    g.payload[rec + 4] = (g.payload[rec + 4].astype(np.int64) * c).astype(np.int32)
    tri = read_triples(g)
    _set64(g.payload, tri, _get64(g.payload, tri) * c)
    return g, lambda check, r: map_result(check, r, value=lambda v: v * c)


def remap_ids(h, base=0):
    """ID_MAP(id + base) for every transfer id; base = 2^29 - k puts ids k - 1 and k + 1 on either side of zero."""
    g = _copy(h)
    rec = transfer_records(g)
    ids = (g.payload[rec + 1].astype(np.int64) << 32) | (g.payload[rec].astype(np.int64) & 0xFFFFFFFF)
    new = ID_MAP(ids + base)
    g.payload[rec] = (new & 0xFFFFFFFF).astype(np.uint32).view(np.int32)
    g.payload[rec + 1] = (new >> 32).astype(np.int32)
    return g, lambda check, r: map_result(check, r, tid=lambda i: ID_MAP(i + base))


def shift_accounts(h):
    d = TOP_ACCOUNT - max_account(h)
    g = _copy(h)
    t = is_transfer(g)
    g.b[t] += d
    g.c[t] += d
    rec = transfer_records(g)
    g.payload[rec + 2] += d
    g.payload[rec + 3] += d
    tri = read_triples(g)
    g.payload[tri] += 2 * d
    return g, lambda check, r: map_result(check, r, key=lambda k: k + 2 * d)


def offsets(keys):
    """offset_counters' per-key constants over sorted keys: +BIG on two keys of every three, -BIG on the third, so the
    sums of 64 or more keys leave int64 and so do the partial sums of keys 32 apart."""
    return {int(k): (-BIG if i % 3 == 2 else BIG) for i, k in enumerate(sorted(keys))}


def wrap_offsets(h):
    """Per-key constants of alternating sign whose total is minus the median read sum of h: keys 32 apart share a sign,
    so the warp's partial sums leave int64, and the low 64 bits of a read's 128-bit sum wrap exactly when its counters
    sum to the median or more.  Only the carry out of the low word orders those reads after the others."""
    tri = read_triples(h)
    keys = sorted(np.unique(h.payload[tri]).tolist())
    out = {k: BIG if i % 2 == 0 else -BIG for i, k in enumerate(keys)}
    ev = np.repeat(np.arange(len(tri) // max(1, len(keys))), len(keys)) if len(keys) else np.zeros(0, np.int64)
    sums = np.bincount(ev, weights=_get64(h.payload, tri).astype(np.float64)) if len(tri) else np.zeros(1)
    out[keys[-1]] -= sum(out.values()) + int(np.median(sums))
    return out


def offset_counters(h, per_key=None):
    g = _copy(h)
    tri = read_triples(g)
    keys = g.payload[tri].astype(np.int64)
    per_key = offsets(np.unique(keys)) if per_key is None else per_key
    lut = np.array([per_key[int(k)] for k in keys], np.int64)
    _set64(g.payload, tri, _get64(g.payload, tri) + lut)

    def expect_mono(check, r):
        assert check == "mono"
        out = map_result(check, r)
        for s in out["shards"]:
            s["edges"] = [(k, kk, v + per_key[kk], v2 + per_key[kk]) if k == abi.MONO_EDGE_MONOTONIC
                          else (k, kk, v, v2) for (k, kk, v, v2) in s["edges"]]
        return out
    return g, expect_mono


TRANSFORMS = {"scale": scale, "remap_ids": remap_ids, "shift_accounts": shift_accounts}


# ---- the checks, by name -------------------------------------------------------------------------------------------
def oracle(check, h, **kw):
    """The library's CPU twin of `check` (its default algorithm)."""
    return {"mono": M.check_monotonic_keys, "cb": M.check_counter_bounds, "tl": M.check_transfer_lookups,
            "rx": M.check_read_explanations, "rg": M.check_read_gaps, "tp": M.check_transfer_placement,
            "sw": M.check_serial_witness}[check](h, **kw)


def device(ctx, check, h, **kw):
    if check == "sw":
        kw.setdefault("witness", True)
    return {"mono": ctx.check_monotonic_keys, "cb": ctx.check_counter_bounds, "tl": ctx.check_transfer_lookups,
            "rx": ctx.check_read_explanations, "rg": ctx.check_read_gaps, "tp": ctx.check_transfer_placement,
            "sw": ctx.check_serial_witness}[check](h, **kw)


def comparable(r):
    """r without its timings, commit_read as a list."""
    out = {k: v for k, v in r.items() if not k.startswith("seconds")}
    if "commit_read" in out:
        out["commit_read"] = np.asarray(out["commit_read"]).tolist()
    return out


# ---- cap shapes ----------------------------------------------------------------------------------------------------
def two(v):
    return {1: (v, 0), 2: (0, v)}


def keys_per_read(nt):
    """Two reads of the same nt keys (accounts 1..ceil(nt/2); account 1's debits nil when nt is odd): one of zeros
    before the ring of :ok unit transfers a -> a + 1 (the last back to 1), one concurrent with them that shows all of
    them.  Every "may" transfer is forced in at the root."""
    A = (nt + 1) // 2
    accts = list(range(1, A + 1))
    dst = {a: a % A + 1 for a in accts}

    def read(p, v):
        ops = [inv_r(p, accts), rd(p, {a: (v, v) for a in accts})]
        if nt % 2:   # a nil counter is left out of the payload
            ops[1]["value"][0][2]["debits-posted"] = None
        return ops
    ops = read(0, 0)
    ops += [tr(a, "invoke", a, dst[a], 1, a) for a in accts]
    ops += read(0, 1)
    ops += [tr(a, "ok", a, dst[a], 1, a) for a in accts]
    return flat(ops)


def units(n, shows, n_ok=None, zeros=0):
    """n unit transfers 1 -> 2 invoked before one read that shows `shows` on both keys, the first n_ok of them
    completing :ok after it and the rest :info (all :ok when n_ok is None); then `zeros` :ok transfers of amount 0.
    With shows = n every transfer is forced in at the root; with shows = 20 all n are free candidates."""
    n_ok = n if n_ok is None else n_ok
    ops = [tr(p, "invoke", 1, 2, 1, p + 1) for p in range(n)]
    ops += [tr(n + 1 + z, "invoke", 1, 2, 0, n + 1 + z) for z in range(zeros)]
    ops += [inv_r(n, [1, 2]), rd(n, two(shows))]
    ops += [tr(p, "ok" if p < n_ok else "info", 1, 2, 1, p + 1) for p in range(n)]
    ops += [tr(n + 1 + z, "ok", 1, 2, 0, n + 1 + z) for z in range(zeros)]
    return flat(ops)


def branching():
    """One read of 9 over :ok transfers 1 -> 2 of 5, 5, 5, 3, 3, 3 concurrent with it: the canonical search takes a 5
    first and must back out of it, so its node count N is a few nodes more than the depth."""
    amounts = [5, 5, 5, 3, 3, 3]
    ops = [tr(p, "invoke", 1, 2, a, p + 1) for p, a in enumerate(amounts)]
    ops += [inv_r(9, [1, 2]), rd(9, two(9))]
    return flat(ops + [tr(p, "ok", 1, 2, a, p + 1) for p, a in enumerate(amounts)])


def placement_chain(k):
    """Reads of 2, 4, ..., 2k one after another, and before the i-th of them an :info transfer of 2: gap 0 holds only
    the first, and each round places one more, so the transfer-placement check needs about k rounds."""
    steps = []
    for i in range(k):
        steps += [("t", f"x{i}", 2), ("r", 2 * (i + 1))]
    return flat(script(steps + [("info", f"x{i}") for i in range(k)])[0])


def witness_chain(k):
    """k :info transfers of 2 invoked first, then reads of 2, 4, ..., 2k: every gap's first solution is the first
    transfer no smaller gap owns, so the witness rounds fix one gap each (k rounds)."""
    steps = [("t", f"x{i}", 2) for i in range(k)] + [("r", 2 * (i + 1)) for i in range(k)]
    return flat(script(steps + [("info", f"x{i}") for i in range(k)])[0])


def int32_max_amounts(extra):
    """Three concurrent :ok transfers 1 -> 2 of INT32_MAX under a read that shows 2 * INT32_MAX + extra."""
    ops = [tr(p, "invoke", 1, 2, INT32_MAX, p + 1) for p in range(3)]
    ops += [inv_r(3, [1, 2]), rd(3, two(2 * INT32_MAX + extra))]
    return flat(ops + [tr(p, "ok", 1, 2, INT32_MAX, p + 1) for p in range(3)])


def zero_amount():
    """An :ok transfer of amount 0 between :ok transfers of 2 and 1 and an :info one of 1, under a read of 3."""
    ops = [tr(0, "invoke", 1, 2, 2, 1), tr(1, "invoke", 1, 2, 0, 2), tr(2, "invoke", 1, 2, 1, 3),
           tr(3, "invoke", 1, 2, 1, 4), inv_r(9, [1, 2]), rd(9, two(3))]
    return flat(ops + [tr(0, "ok", 1, 2, 2, 1), tr(1, "ok", 1, 2, 0, 2), tr(2, "ok", 1, 2, 1, 3),
                       tr(3, "info", 1, 2, 1, 4)])


def _one_read(v):
    return flat([inv_r(0, [1, 2]), rd(0, two(v))])


def _torn():
    """Two reads that disagree with the one transfer between them (KEY in K10-K12)."""
    return flat([tr(0, "invoke", 1, 2, 3, 1), tr(0, "ok", 1, 2, 3, 1), inv_r(1, [1, 2]), rd(1, {1: (3, 0), 2: (0, 2)})])


def many_shards(n):
    """n shards: most hold one read and no transfer; every 97th a transfer and a read it explains, every 1001st a read
    that contradicts its transfer (so the witness is chosen among many reads of many shards)."""
    kinds = {"read": _one_read(0), "ok": units(1, 1), "torn": _torn()}
    parts = [kinds["torn"] if s % 1001 == 500 else kinds["ok"] if s % 97 == 3 else kinds["read"] for s in range(n)]
    return H.concat_keys(parts)
