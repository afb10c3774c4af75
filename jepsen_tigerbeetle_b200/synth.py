"""Deterministic synthetic Jepsen histories for the BASELINE.json configs (SURVEY §8(d)).

Counter-based RNG (splitmix64 seeding a PCG32 stream) so the same (config, seed) gives the same
history everywhere.  Per client thread: invoke, Exp(tau_op) duration, a linearization point uniform
inside the op's interval; all linearization points are sorted and applied to the true model to get
return values, so every generated history is linearizable by construction ("valid" variants).
`stale_read` then makes one ok read return an old state (ground truth is decided by the oracle).

Op shapes follow the reference generators:
  set-full   adds/reads 1:1 over random keys      set_full.clj:22-45,159
  bank       reads of all accounts / transfers    tests/ledger.clj:27-67 (amount 1..max-transfer, debit != credit)
  :info      client timeouts                      set_full.clj:107-110 ; workloads/ledger.clj:46-48
             after an :info the thread continues as process + concurrency (jepsen convention)
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from .history import (F_ADD, F_CAS, F_LOOKUP, F_READ, F_TRANSFER, F_WRITE, FLAG_FINAL, NIL, T_FAIL, T_INFO,
                      T_INVOKE, T_OK, TRANSFER_RECORD, FlatHistory)

MASK64 = (1 << 64) - 1


class PCG32:
    """PCG-XSH-RR 64/32 seeded through splitmix64."""

    def __init__(self, seed: int, stream: int = 0) -> None:
        x = (seed * 0x9E3779B97F4A7C15 + stream) & MASK64
        self._sm = x
        self.state = 0
        self.inc = ((self._splitmix() << 1) | 1) & MASK64
        self.state = (self._splitmix() + self.inc) & MASK64
        self.u32()

    def _splitmix(self) -> int:
        self._sm = (self._sm + 0x9E3779B97F4A7C15) & MASK64
        z = self._sm
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
        return z ^ (z >> 31)

    def u32(self) -> int:
        old = self.state
        self.state = (old * 6364136223846793005 + self.inc) & MASK64
        xorshifted = (((old >> 18) ^ old) >> 27) & 0xFFFFFFFF
        rot = old >> 59
        return ((xorshifted >> rot) | (xorshifted << ((-rot) & 31))) & 0xFFFFFFFF

    def below(self, n: int) -> int:
        """Uniform integer in [0, n) (n < 2**32), multiply-shift."""
        return (self.u32() * n) >> 32

    def unit(self) -> float:
        """Uniform double in (0, 1]."""
        return (self.u32() + 1) / 4294967296.0

    def exp_ns(self, mean_ns: float) -> int:
        return max(2, int(-mean_ns * math.log(self.unit())))


@dataclass
class SynthSpec:
    model: str                   # 'register' | 'cas-register' | 'set' | 'bank'
    n_ops: int
    n_clients: int
    seed: int = 1
    p_info: float = 0.0
    n_keys: int = 1
    grouped_keys: bool = False   # True: threads partitioned over keys (independent/concurrent-generator)
    tau_op_ns: float = 10e6
    tau_think_ns: float = 0.0
    n_values: int = 5            # register values 0..n_values-1
    n_accounts: int = 8          # bank accounts 1..8 (core.clj:208-210)
    max_transfer: int = 5        # tests/ledger.clj:355
    first_element: int = 9       # set_full.clj:159: adds start after the pre-created accounts
    stale_read: bool = False     # make one ok read stale ("invalid" variant; oracle decides)
    stale_frac: float = 0.9
    stale_by: int = 0            # linearization steps back (0 => 8 * clients-per-key)
    final_reads: bool = False    # quiesce + one :final? read per key (set_full.clj:161-170)


def generate(spec: SynthSpec) -> FlatHistory:
    return _generate(spec)


def generate_ledger_counters(spec: SynthSpec, fractured: bool = False, lost_transfer: bool = False,
                             duplicated_transfer: bool = False) -> FlatHistory:
    """The ledger-counter form of a bank `spec` (what flatten_ops(..., "ledger-counters") makes of a ledger history):
    the same events as generate(spec), but every :ok read carries each account's debits-posted and credits-posted
    as (key, value_lo, value_hi) triples, key = 2 * account + field, and credits - debits is the balance generate(spec)
    reports.  `spec.stale_read` makes the same read stale as in generate(spec).  fractured=True instead takes ONE account
    of one read from an older snapshot (a "fractured read"; the oracle decides the ground truth).  `spec.final_reads`
    adds one quiesced :final? read per key that returns the final counters.
    lost_transfer=True never applies the counters of one :ok transfer; duplicated_transfer=True applies them twice.  The
    transfer is the middle one, in linearization order, of the :ok transfers of key 0 (no extra random draws, so the
    events and every other value equal the unmutated history); its op number is meta["lost_op_index"] /
    meta["duplicated_op_index"]."""
    if spec.model != "bank":
        raise ValueError("the ledger-counter form needs a bank spec")
    if lost_transfer and duplicated_transfer:
        raise ValueError("lost_transfer and duplicated_transfer are exclusive")
    return _generate(spec, counters=True, fracture=fractured, lost=lost_transfer, duplicated=duplicated_transfer)


def generate_ledger_lookups(spec: SynthSpec, p_lookup: float = 0.0, lost_transfer: bool = False,
                            phantom_record: bool = False, mismatched_record: bool = False,
                            vanished_record: bool = False, inflated_read: bool = False, torn_transfer: bool = False,
                            torn_pair: bool = False, split_amount: bool = False) -> FlatHistory:
    """The ledger-lookups form of a one-key bank `spec` (what flatten_ops(..., "ledger-lookups") makes of a ledger
    history): the events of generate_ledger_counters(spec), every transfer invoke carrying its record (id, debit,
    credit, amount) with ids 1, 2, ... in invocation order, then one quiesced :final? lookup per client, one after
    another, each returning every committed transfer (the :ok ones and the :info ones that took effect) in id order.
    p_lookup > 0 (small histories only) adds about p_lookup * n_ops mid-history lookups, each on a process of its own,
    drawn from a second random stream; each returns the committed transfers linearized before a point inside its
    interval, and every event's :index is then its position.
    Mutations (no extra random draws; several may be combined):
      lost_transfer      generate_ledger_counters' lost transfer, missing from every lookup as well (LOST)
      phantom_record     the first final lookup also returns an id no transfer carries (PHANTOM)
      mismatched_record  the first final lookup returns its middle record with amount + 1 (MISMATCH)
      vanished_record    the last final lookup drops the middle committed :info transfer (VANISHED, and the final
                         read, which completes first, now lies above that lookup's sums; needs p_info > 0 and two
                         clients)
      inflated_read      the final read's first counter is one more than it was (READ_ABOVE_LOOKUP; needs
                         spec.final_reads)
    Read mutations for the read-explanation check (the first non-final :ok read, from the middle of the history on,
    that has what the mutation needs among the :ok transfers concurrent with it; meta["torn_read_index"] is its :index):
      torn_transfer      the read shows only the debit half of one concurrent transfer
      torn_pair          two concurrent transfers of equal amount on four distinct accounts: the read shows the debit
                         half of the first and the credit half of the second, so the totals still hold
      split_amount       the read shows amount - 1 of a concurrent transfer (amount >= 2) on both sides"""
    if spec.model != "bank" or spec.n_keys != 1:
        raise ValueError("the ledger-lookups form needs a one-key bank spec")
    if inflated_read and not spec.final_reads:
        raise ValueError("inflated_read needs spec.final_reads")
    ex: dict = {}
    base = _generate(spec, counters=True, lost=lost_transfer, extra=ex)
    ops, op_ev, C = ex["ops"], ex["op_of_event"], spec.n_clients
    n = base.n_events
    # ---- transfer records: ids 1, 2, ... in invocation order ----------------------------------------------------
    tin = np.nonzero((base.f == F_TRANSFER) & (base.type == T_INVOKE))[0]
    t_ops = op_ev[tin]
    o_arr = np.array([ops[i] for i in t_ops], np.int64).reshape(-1, 11)
    ids = np.arange(1, len(tin) + 1, dtype=np.int64)
    rec = np.zeros((len(tin), TRANSFER_RECORD), np.int32)
    rec[:, 0], rec[:, 2], rec[:, 3], rec[:, 4] = ids, o_arr[:, 8], o_arr[:, 9], o_arr[:, 7]
    committed = o_arr[:, 10] < 2
    if lost_transfer and ex["mutated_transfer"] >= 0:
        committed &= t_ops != ex["mutated_transfer"]
    t_lin = o_arr[:, 2]
    # ---- lookups: (time, process, records) ----------------------------------------------------------------------
    lookups: list[tuple[int, int, int, np.ndarray, bool]] = []   # (invoke time, completion time, process, recs, final)
    max_proc = int(base.process.max()) if n else -1
    if p_lookup > 0 and n:
        rng = PCG32(spec.seed, 2)
        t0, t1 = int(base.time_ns[0]), int(base.time_ns[~(base.flags & FLAG_FINAL).astype(bool)].max())
        for j in range(int(round(p_lookup * spec.n_ops))):
            q = t0 + 1 + rng.below(max(1, t1 - t0))
            lookups.append((q - rng.exp_ns(spec.tau_op_ns), q + rng.exp_ns(spec.tau_op_ns), max_proc + 1 + j,
                            rec[committed & (t_lin < q)], False))
    tq = int(base.time_ns.max()) + 1_000_000_000 if n else 0
    last_proc = list(range(C))
    for p in np.unique(base.process):
        last_proc[int(p) % C] = max(last_proc[int(p) % C], int(p))
    fin = rec[committed]
    for t in range(C):
        lookups.append((tq + 2 * t, tq + 2 * t + 1, last_proc[t], fin, True))
    n_final = C
    finals = [i for i, lk in enumerate(lookups) if lk[4]]
    if phantom_record:
        i = finals[0]
        extra = fin[len(fin) // 2].copy() if len(fin) else np.array([0, 0, 1, 2, 1], np.int32)
        extra[0], extra[1] = len(tin) + 1, 0
        lookups[i] = lookups[i][:3] + (np.concatenate([lookups[i][3], extra[None]]),) + lookups[i][4:]
    if mismatched_record:
        i = finals[0]
        r = lookups[i][3].copy()
        r[len(r) // 2, 4] += 1
        lookups[i] = lookups[i][:3] + (r,) + lookups[i][4:]
    if vanished_record:
        info = np.nonzero(committed & (o_arr[:, 10] == 1))[0]
        if len(info) == 0 or n_final < 2:
            raise ValueError("vanished_record needs a committed :info transfer and two clients")
        gone = ids[info[len(info) // 2]]
        i = finals[-1]
        lookups[i] = lookups[i][:3] + (lookups[i][3][lookups[i][3][:, 0] != gone],) + lookups[i][4:]
    # ---- events, payload ----------------------------------------------------------------------------------------
    L = len(lookups)
    plen_pre = np.concatenate([base.payload_len, np.full(2 * L, -1, np.int32)])
    plen_pre[tin] = TRANSFER_RECORD
    for j, lk in enumerate(lookups):
        plen_pre[n + 2 * j + 1] = lk[3].size
    lens = np.maximum(plen_pre, 0).astype(np.int64)
    poff_pre = np.zeros(n + 2 * L, np.int64)
    np.cumsum(lens[:-1], out=poff_pre[1:])
    payload = np.zeros(int(lens.sum()), np.int32)
    reads = np.nonzero(base.payload_len > 0)[0]
    if len(reads):
        rl = base.payload_len[reads].astype(np.int64)
        within = np.arange(int(rl.sum())) - np.repeat(np.cumsum(rl) - rl, rl)
        payload[np.repeat(poff_pre[reads], rl) + within] = base.payload[np.repeat(base.payload_off[reads], rl) + within]
    payload[poff_pre[tin][:, None] + np.arange(TRANSFER_RECORD)] = rec
    for j, lk in enumerate(lookups):
        o = poff_pre[n + 2 * j + 1]
        payload[o:o + lk[3].size] = lk[3].reshape(-1)
    if inflated_read:
        e = np.nonzero((base.flags & FLAG_FINAL).astype(bool) & (base.type == T_OK) & (base.f == F_READ))[0][0]
        payload[poff_pre[e] + 1] += 1
    torn_at = -1
    for kind in [k for k, on in (("transfer", torn_transfer), ("pair", torn_pair), ("split", split_amount)) if on]:
        torn_at = _tear_read(kind, base, ops, op_ev, ex["mutated_transfer"], payload, poff_pre)
    lt = np.array([x for lk in lookups for x in lk[:2]], np.int64)
    time_pre = np.concatenate([base.time_ns, lt])
    order = np.argsort(time_pre, kind="stable")
    cat = lambda arr, tail: np.concatenate([arr, np.asarray(tail, arr.dtype)])[order]   # noqa: E731
    typ = cat(base.type, [T_INVOKE, T_OK] * L)
    f = cat(base.f, [F_LOOKUP] * (2 * L))
    flags = cat(base.flags, [FLAG_FINAL if lk[4] else 0 for lk in lookups for _ in (0, 1)])
    proc = cat(base.process, [lk[2] for lk in lookups for _ in (0, 1)])
    zeros = [0] * (2 * L)
    index = (cat(base.index, np.arange(n, n + 2 * L)) if p_lookup <= 0 else
             np.arange(n + 2 * L, dtype=np.int32))
    meta = dict(base.meta, model="ledger-lookups", n_ops=base.meta["n_ops"] + L, multi_transfer_txns=0,
                n_lookups=L)
    if torn_transfer or torn_pair or split_amount:
        meta["torn_read_index"] = int(index[np.nonzero(order == torn_at)[0][0]])
    h = FlatHistory(typ, f, flags, proc, index.astype(np.int32), time_pre[order], cat(base.a, zeros),
                    cat(base.b, zeros), cat(base.c, zeros), poff_pre[order], plen_pre[order], payload,
                    np.array([0, n + 2 * L], np.int64), base.key_ids.copy(), meta)
    h.validate()
    return h


def _tear_read(kind: str, base: FlatHistory, ops: list, op_ev: np.ndarray, skip: int, payload: np.ndarray,
               poff: np.ndarray) -> int:
    """One read mutation of generate_ledger_lookups (no random draws) on the payload of the lookups form; returns the
    base event of the read.  A read's payload is (2a, debits, 0, 2a + 1, credits, 0) per account a = 1, 2, ..."""
    reads = np.nonzero((base.f == F_READ) & (base.type == T_OK) & ~(base.flags & FLAG_FINAL).astype(bool))[0]
    reads = np.concatenate([reads[len(reads) // 2:], reads[:len(reads) // 2]])
    tr = [i for i, o in enumerate(ops) if o[6] == F_TRANSFER and o[10] == 0 and i != skip]
    t_inv = np.array([ops[i][0] for i in tr], np.int64)
    t_ret = np.array([ops[i][1] for i in tr], np.int64)

    def add(e: int, acct: int, field: int, x: int) -> None:
        payload[poff[e] + 6 * (acct - 1) + 3 * field + 1] += x

    for e in reads:
        r = ops[op_ev[e]]
        conc = [tr[j] for j in np.nonzero((t_inv < r[1]) & (t_ret > r[0]))[0]]
        seen = lambda i: ops[i][2] < r[2]   # noqa: E731  (linearized before the read)
        if kind == "transfer" and conc:
            t = ops[conc[0]]
            if seen(conc[0]):
                add(e, t[9], 1, -t[7])
            else:
                add(e, t[8], 0, t[7])
            return int(e)
        if kind == "split":
            big = [i for i in conc if ops[i][7] >= 2]
            if big:
                t = ops[big[0]]
                x = -1 if seen(big[0]) else t[7] - 1
                add(e, t[8], 0, x)
                add(e, t[9], 1, x)
                return int(e)
        if kind == "pair":
            for a in range(len(conc)):
                for b in range(a + 1, len(conc)):
                    t1, t2 = ops[conc[a]], ops[conc[b]]
                    if t1[7] != t2[7] or {t1[8], t1[9]} & {t2[8], t2[9]}:
                        continue
                    if seen(conc[a]):
                        add(e, t1[9], 1, -t1[7])
                    else:
                        add(e, t1[8], 0, t1[7])
                    if seen(conc[b]):
                        add(e, t2[8], 0, -t2[7])
                    else:
                        add(e, t2[9], 1, t2[7])
                    return int(e)
    raise ValueError(f"no read has what the {kind} mutation needs")


def _generate(spec: SynthSpec, counters: bool = False, fracture: bool = False, lost: bool = False,
              duplicated: bool = False, extra: dict | None = None) -> FlatHistory:
    rng = PCG32(spec.seed, 1)
    C, K = spec.n_clients, spec.n_keys
    model = spec.model
    # ---- phase 1: op intervals per thread -------------------------------------------------------
    next_inv = [0] * C
    for t in range(C):
        next_inv[t] = 1 + t  # staggered by 1 ns so the first invokes have a defined order
    proc = list(range(C))
    ops = []  # dicts are slow; use tuples: (t_inv, t_ret, t_lin, thread, process, key, f, a, b, c, fate)
    next_elem = spec.first_element
    import heapq
    heap = [(next_inv[t], t) for t in range(C)]
    heapq.heapify(heap)
    per_key_threads = max(1, C // K) if spec.grouped_keys else C
    for _ in range(spec.n_ops):
        t_inv, t = heapq.heappop(heap)
        dur = rng.exp_ns(spec.tau_op_ns)
        t_ret = t_inv + dur
        t_lin = t_inv + 1 + rng.below(max(1, min(dur - 1, 0xFFFFFFFF)))
        if spec.grouped_keys:
            key = min(K - 1, t // per_key_threads)
        else:
            key = rng.below(K) if K > 1 else 0
        a = b = c = 0
        if model in ("register", "cas-register"):
            kind = rng.below(3 if model == "cas-register" else 2)
            if kind == 0:
                f = F_READ
            elif kind == 1:
                f, a = F_WRITE, rng.below(spec.n_values)
            else:
                f, a, b = F_CAS, rng.below(spec.n_values), rng.below(spec.n_values)
        elif model == "set":
            if rng.below(2) == 0:
                f, a = F_ADD, next_elem
                next_elem += 1
            else:
                f = F_READ
        elif model == "bank":
            if rng.below(2) == 0:
                f = F_READ
            else:
                f = F_TRANSFER
                b = 1 + rng.below(spec.n_accounts)
                c = 1 + rng.below(spec.n_accounts - 1)
                if c >= b:
                    c += 1
                a = 1 + rng.below(spec.max_transfer)
        else:
            raise ValueError(model)
        fate = 0  # 0 ok, 1 info+applied, 2 info+not applied
        if spec.p_info > 0 and rng.unit() <= spec.p_info:
            fate = 1 if rng.below(2) == 0 else 2
        ops.append([t_inv, t_ret, t_lin, t, proc[t], key, f, a, b, c, fate])
        if fate:
            proc[t] += C
        think = rng.exp_ns(spec.tau_think_ns) if spec.tau_think_ns > 0 else 1
        heapq.heappush(heap, (t_ret + think, t))
    # ---- phase 2: apply in linearization order --------------------------------------------------
    order = sorted(range(len(ops)), key=lambda i: (ops[i][2], i))
    reg = [NIL] * K
    bal = [[0] * spec.n_accounts for _ in range(K)]
    sets: list[list[int]] = [[] for _ in range(K)]
    results: list = [None] * len(ops)   # read values / cas success
    snapshots: list[list] = [[] for _ in range(K)]  # per key: state snapshots per lin step (for stale reads)
    lin_pos = [0] * len(ops)
    want_snap = spec.stale_read or fracture
    # ledger-counter form: per key and account the two counters that only grow, per read their values
    debits = [[0] * spec.n_accounts for _ in range(K)]
    credits = [[0] * spec.n_accounts for _ in range(K)]
    cresults: list = [None] * len(ops)
    csnapshots: list[list] = [[] for _ in range(K)]
    # the :ok transfer whose counters are applied 0 or 2 times (lost / duplicated), -1 = none
    mutated_transfer = -1
    if lost or duplicated:
        cand = [i for i in order if ops[i][6] == F_TRANSFER and ops[i][10] == 0 and ops[i][5] == 0]
        if cand:
            mutated_transfer = cand[len(cand) // 2]
    for i in order:
        (_ti, _tr, _tl, _t, _p, key, f, a, b, c, fate) = ops[i]
        if want_snap:
            lin_pos[i] = len(snapshots[key])
            if model in ("register", "cas-register"):
                snapshots[key].append(reg[key])
            elif model == "bank":
                snapshots[key].append(tuple(bal[key]))
                if counters:
                    csnapshots[key].append((tuple(debits[key]), tuple(credits[key])))
            else:
                snapshots[key].append(len(sets[key]))
        if fate == 2:
            continue
        if f == F_READ:
            if model in ("register", "cas-register"):
                results[i] = reg[key]
            elif model == "bank":
                results[i] = tuple(bal[key])
                if counters:
                    cresults[i] = (tuple(debits[key]), tuple(credits[key]))
            else:
                results[i] = len(sets[key])  # prefix length of sets[key] in lin order
        elif f == F_WRITE:
            reg[key] = a
        elif f == F_CAS:
            if reg[key] == a:
                reg[key] = b
                results[i] = True
            else:
                results[i] = False
        elif f == F_ADD:
            sets[key].append(a)
        elif f == F_TRANSFER:
            bal[key][b - 1] -= a
            bal[key][c - 1] += a
            if counters:
                times = 1 if i != mutated_transfer else 0 if lost else 2
                debits[key][b - 1] += times * a
                credits[key][c - 1] += times * a
    # ---- stale-read mutation --------------------------------------------------------------------
    mutated = -1
    if spec.stale_read:
        cand = [i for i in sorted(range(len(ops)), key=lambda i: ops[i][1])
                if ops[i][6] == F_READ and ops[i][10] == 0 and ops[i][5] == 0]
        if cand:
            back = spec.stale_by or 8 * per_key_threads
            start = int(spec.stale_frac * len(cand))
            for i in cand[start:] + cand[:start][::-1]:
                key = ops[i][5]
                p = max(0, lin_pos[i] - back)
                old = snapshots[key][p]
                if old != results[i] and not (model == "set" and old >= results[i]):
                    results[i] = old
                    if counters:
                        cresults[i] = csnapshots[key][p]
                    mutated = i
                    break
    fractured_at = -1
    if fracture:
        cand = [i for i in sorted(range(len(ops)), key=lambda i: ops[i][1])
                if ops[i][6] == F_READ and ops[i][10] == 0 and ops[i][5] == 0]
        back = spec.stale_by or 8 * per_key_threads
        start = int(spec.stale_frac * len(cand))
        for i in cand[start:] + cand[:start][::-1]:
            old_d, old_c = csnapshots[ops[i][5]][max(0, lin_pos[i] - back)]
            cur_d, cur_c = cresults[i]
            changed = [j for j in range(spec.n_accounts) if (old_d[j], old_c[j]) != (cur_d[j], cur_c[j])]
            if changed:
                j = changed[0]
                cresults[i] = (cur_d[:j] + (old_d[j],) + cur_d[j + 1:], cur_c[:j] + (old_c[j],) + cur_c[j + 1:])
                fractured_at = i
                break
    # ---- phase 3: events ------------------------------------------------------------------------
    ev = []  # (time, seq, op, is_completion)
    for i, o in enumerate(ops):
        ev.append((o[0], 0, i, 0))
        ev.append((o[1], 1, i, 1))
    t_end = max(o[1] for o in ops) if ops else 0
    final_ops = []
    if spec.final_reads:
        # quiesce 5 s then one final read per key on thread 0.. (set_full.clj:161-170)
        tq = t_end + 5_000_000_000
        for key in range(K):
            i = len(ops) + len(final_ops)
            final_ops.append([tq + 2 * key, tq + 2 * key + 1, 0, key % C, proc[key % C], key,
                              F_READ, 0, 0, 0, 0])
            ev.append((tq + 2 * key, 0, i, 0))
            ev.append((tq + 2 * key + 1, 1, i, 1))
    ev.sort()
    all_ops = ops + final_ops
    n = len(ev)
    typ = np.zeros(n, np.uint8); f_arr = np.zeros(n, np.uint8); flags = np.zeros(n, np.uint8)
    proc_arr = np.zeros(n, np.int32); idx = np.arange(n, dtype=np.int32)
    time_arr = np.zeros(n, np.int64)
    a_arr = np.zeros(n, np.int32); b_arr = np.zeros(n, np.int32); c_arr = np.zeros(n, np.int32)
    plen = np.zeros(n, np.int32)
    keys_arr = np.zeros(n, np.int64)
    payload_chunks: list[np.ndarray] = [None] * n  # type: ignore[list-item]
    sets_np = [np.array(s, dtype=np.int32) for s in sets]
    empty = np.zeros(0, np.int32)
    acct_ids = np.arange(1, spec.n_accounts + 1, dtype=np.int32)
    for e, (tm, _seq, i, comp) in enumerate(ev):
        o = all_ops[i]
        is_final = i >= len(ops)
        f = o[6]
        time_arr[e] = tm; proc_arr[e] = o[4]; f_arr[e] = f; keys_arr[e] = o[5]
        a_arr[e], b_arr[e], c_arr[e] = o[7], o[8], o[9]
        payload_chunks[e] = empty
        if is_final:
            flags[e] = 1
        if not comp:
            typ[e] = T_INVOKE
            if f == F_READ:
                a_arr[e] = NIL
                plen[e] = -1
            continue
        fate = o[10]
        if fate:
            typ[e] = T_INFO
            if f == F_READ:
                a_arr[e] = NIL
                plen[e] = -1
            continue
        typ[e] = T_OK
        if f == F_CAS and not results[i]:
            typ[e] = T_FAIL
        elif f == F_READ:
            if model in ("register", "cas-register"):
                a_arr[e] = results[i]
            elif model == "bank" and counters:
                d, cr = (tuple(debits[o[5]]), tuple(credits[o[5]])) if is_final else cresults[i]
                pl = np.zeros((spec.n_accounts, 2, 3), np.int64)
                pl[:, 0, 0] = 2 * acct_ids
                pl[:, 1, 0] = 2 * acct_ids + 1
                pl[:, 0, 1] = d
                pl[:, 1, 1] = cr   # counters of synthetic histories stay far below 2^31: value_hi = 0
                payload_chunks[e] = pl.reshape(-1).astype(np.int32)
                plen[e] = 6 * spec.n_accounts
            elif model == "bank":
                r = results[i]
                pl = np.empty(2 * spec.n_accounts, np.int32)
                pl[0::2] = acct_ids
                pl[1::2] = r
                payload_chunks[e] = pl
                plen[e] = pl.shape[0]
            else:
                k = o[5]
                cnt = len(sets[k]) if is_final else results[i]
                pl = np.sort(sets_np[k][:cnt])
                payload_chunks[e] = pl
                plen[e] = cnt
    # ---- CSR by key ------------------------------------------------------------------------------
    perm = np.argsort(keys_arr, kind="stable")
    counts = np.bincount(keys_arr.astype(np.int64), minlength=K)
    shard_off = np.zeros(K + 1, np.int64)
    np.cumsum(counts, out=shard_off[1:])
    plen_p = plen[perm]
    lens = np.maximum(plen_p, 0).astype(np.int64)
    poff = np.zeros(n, np.int64)
    if n:
        np.cumsum(lens[:-1], out=poff[1:])
    chunks = [payload_chunks[j] for j in perm]
    payload = np.concatenate(chunks).astype(np.int32) if chunks else empty
    meta = {"model": "ledger-counters" if counters else model, "spec": spec, "mutated_op_index": mutated,
            "n_ops": len(all_ops), "accounts": list(range(1, spec.n_accounts + 1))}
    if counters:
        meta["fractured_op_index"] = fractured_at
        if lost:
            meta["lost_op_index"] = mutated_transfer
        if duplicated:
            meta["duplicated_op_index"] = mutated_transfer
    if extra is not None:   # what generate_ledger_lookups builds on
        extra.update(ops=all_ops, op_of_event=np.array([e[2] for e in ev], np.int64)[perm],
                     mutated_transfer=mutated_transfer)
    h = FlatHistory(typ[perm], f_arr[perm], flags[perm], proc_arr[perm], idx[perm], time_arr[perm],
                    a_arr[perm], b_arr[perm], c_arr[perm], poff, plen_p, payload, shard_off,
                    np.arange(1, K + 1, dtype=np.int64), meta)
    h.validate()
    return h


# ---- the five BASELINE.json configs (SURVEY §8(d)) ---------------------------------------------
def config_c1(seed: int = 1, **kw) -> FlatHistory:
    """set-full :linearizable? true, 100 ops, 4 clients, 1 key."""
    return generate(SynthSpec("set", 100, 4, seed, final_reads=True, **kw))


def config_c2(seed: int = 1, p_info: float = 0.0, **kw) -> FlatHistory:
    """1k-op cas-register history, 16 concurrent clients."""
    return generate(SynthSpec("cas-register", 1000, 16, seed, p_info=p_info, **kw))


def config_c3(seed: int = 1, p_info: float = 0.0, **kw) -> FlatHistory:
    """10k-op bank-transfer history, 32 clients (headline)."""
    return generate(SynthSpec("bank", 10000, 32, seed, p_info=p_info, **kw))


def config_c4(seed: int = 1, n_keys: int = 64, p_info: float = 0.01, n_ops: int = 100000,
              **kw) -> FlatHistory:
    """100k-op set-full grow-only history, 64 clients, K ledgers."""
    return generate(SynthSpec("set", n_ops, 64, seed, p_info=p_info, n_keys=n_keys,
                              final_reads=True, **kw))


def config_c5(seed: int = 1, n_keys: int = 256, p_info: float = 0.30, n_ops: int = 50000,
              **kw) -> FlatHistory:
    """50k-op adversarial cas-register history, 30% :info, 8 clients per key."""
    return generate(SynthSpec("cas-register", n_ops, 8 * n_keys, seed, p_info=p_info,
                              n_keys=n_keys, grouped_keys=True, **kw))


def poison_c5(h: FlatHistory, shard: int = 7) -> FlatHistory:
    """One key of a C5 history made non-linearizable: its third :ok read returns a value nobody ever wrote
    (values are 0..4).  The merged verdict of the keyed check must flip to invalid with exactly one failure."""
    import copy
    from . import history as H
    h = copy.deepcopy(h)
    lo, hi = int(h.shard_off[shard]), int(h.shard_off[shard + 1])
    reads = [e for e in range(lo, hi) if h.f[e] == H.F_READ and h.type[e] == H.T_OK]
    h.a[reads[min(2, len(reads) - 1)]] = 99
    return h


def poison_c4(h: FlatHistory, shard: int = 5) -> FlatHistory:
    """One ledger of a C4 history loses elements: the two largest ids vanish from the ledger's LAST non-final :ok read
    (payloads are sorted), so elements a read has already seen are :lost -> set-full invalid for that ledger."""
    import copy
    from . import history as H
    h = copy.deepcopy(h)
    lo, hi = int(h.shard_off[shard]), int(h.shard_off[shard + 1])
    reads = [e for e in range(lo, hi) if h.f[e] == H.F_READ and h.type[e] == H.T_OK and h.payload_len[e] > 4
             and not (h.flags[e] & 1)]
    h.payload_len[reads[-1]] -= 2
    return h
