"""ctypes images of the result/option structs in include/jtb_check.h (keep in lock-step)."""
from __future__ import annotations

import ctypes as C

from .history import MAX_ACCOUNTS, CHistory

ABI_VERSION = 10
OPT_NO_EAGER_READS = 1
OPT_NO_SCOUTS = 2
OPT_ENGINE_LEVEL = 4
OPT_ENGINE_WORKLIST = 8
OPT_NO_BEAM = 16

CAUSE_NONE, CAUSE_TABLE_FULL, CAUSE_BUDGET, CAUSE_TOO_WIDE, CAUSE_PARTIAL_READ = 0, 1, 2, 3, 4
CAUSE_ANOMALY, CAUSE_UNDECIDED, CAUSE_NO_WITNESS, CAUSE_REAL_TIME = 5, 6, 7, 8
CAUSE_NAME = {0: None, 1: "table-full", 2: "budget", 3: "too-wide", 4: "partial-read", 5: "anomaly", 6: "undecided",
              7: "no-witness", 8: "real-time", 9: "lookup"}
MONO_NO_REALTIME = 1
MONO_EDGE_NONE, MONO_EDGE_MONOTONIC, MONO_EDGE_REALTIME = 0, 1, 2
CB_BELOW, CB_ABOVE = 1, 2
(TL_PHANTOM, TL_MISMATCH, TL_FAILED_VISIBLE, TL_FUTURE, TL_DUPLICATE, TL_LOST, TL_VANISHED, TL_READ_BELOW_LOOKUP,
 TL_READ_ABOVE_LOOKUP) = range(1, 10)
TL_KINDS = 9
TL_KIND_NAME = {1: "phantom", 2: "mismatch", 3: "failed-visible", 4: "future", 5: "duplicate", 6: "lost",
                7: "vanished", 8: "read-below-lookup", 9: "read-above-lookup"}
RX_KEY, RX_JOINT = 1, 2
RX_KIND_NAME = {1: "key", 2: "joint"}
RX_MAX_KEYS, RX_MAX_GATHER, RX_MAX_FREE, RX_DEFAULT_MAX_NODES = 256, 128, 64, 4096
RG_KEY, RG_JOINT, RG_DOUBLE = 1, 2, 3
RG_KIND_NAME = {1: "key", 2: "joint", 3: "double"}
RG_MAX_KEYS, RG_MAX_GATHER, RG_MAX_FREE, RG_DEFAULT_MAX_NODES = 256, 128, 64, 4096
TP_KEY, TP_JOINT, TP_DOUBLE, TP_LOST = 1, 2, 3, 4
TP_KIND_NAME = {1: "key", 2: "joint", 3: "double", 4: "lost"}
TP_MAX_KEYS, TP_MAX_GATHER, TP_MAX_FREE, TP_DEFAULT_MAX_NODES = RG_MAX_KEYS, RG_MAX_GATHER, RG_MAX_FREE, 4096
TP_DEFAULT_MAX_ROUNDS = 64
SW_NEVER, SW_AFTER, SW_FREE = -1, -2, -3
SF_NEVER_READ, SF_STABLE, SF_LOST = 0, 1, 2
BANK_OK, BANK_UNEXPECTED_KEY, BANK_NIL_BALANCE, BANK_WRONG_TOTAL, BANK_NEGATIVE_VALUE = range(5)
BANK_ERR_NAME = {1: "unexpected-key", 2: "nil-balance", 3: "wrong-total", 4: "negative-value"}


class COpts(C.Structure):
    _fields_ = [("device", C.c_int32), ("flags", C.c_int32), ("table_bytes", C.c_uint64),
                ("max_configs", C.c_uint64), ("time_budget_ms", C.c_uint32),
                ("search_ctas", C.c_uint32)]


class CLinShard(C.Structure):
    _fields_ = [("valid", C.c_int32), ("witness_index", C.c_int32),
                ("previous_ok_index", C.c_int32), ("cause", C.c_int32),
                ("configs_explored", C.c_uint64), ("probes", C.c_uint64)]


class CFinalConfig(C.Structure):
    """jtb_final_config: one of knossos' :configs of an INVALID shard."""
    _fields_ = [("state", C.c_int32), ("balances", C.c_int32 * MAX_ACCOUNTS), ("n_pending", C.c_int32),
                ("n_linearized_open", C.c_int32), ("n_crashed_linearized", C.c_int32),
                ("pending_index", C.c_int32 * 64), ("linearized_open_index", C.c_int32 * 64)]


def final_configs_to_list(buf, n: int) -> list[dict]:
    return [{"state": c.state, "balances": list(c.balances),
             "pending": list(c.pending_index[:c.n_pending]),
             "linearized_open": list(c.linearized_open_index[:c.n_linearized_open]),
             "crashed_linearized": c.n_crashed_linearized} for c in buf[:n]]


class CLinResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32),
                ("configs_explored", C.c_uint64), ("probes", C.c_uint64),
                ("hbm_bytes_algorithmic", C.c_uint64), ("key_bytes", C.c_uint32),
                ("reserved0", C.c_uint32), ("seconds_kernel", C.c_double),
                ("seconds_total", C.c_double)]


class CSetFullShard(C.Structure):
    _fields_ = [("valid", C.c_int32), ("attempt_count", C.c_int32), ("stable_count", C.c_int32),
                ("lost_count", C.c_int32), ("never_read_count", C.c_int32),
                ("stale_count", C.c_int32), ("duplicated_count", C.c_int32),
                ("suspect_final_reads", C.c_int32), ("stable_latency_max_ms", C.c_int64),
                ("lost_latency_max_ms", C.c_int64)]


class CSetFullOut(C.Structure):
    _fields_ = [("shards", C.c_void_p), ("elem_capacity", C.c_int64), ("elem_off", C.c_void_p),
                ("elem_id", C.c_void_p), ("elem_outcome", C.c_void_p),
                ("elem_latency_ms", C.c_void_p), ("elem_dup_count", C.c_void_p),
                ("valid", C.c_int32), ("n_failures", C.c_int32), ("seconds_kernel", C.c_double),
                ("seconds_total", C.c_double),
                ("suspect_capacity", C.c_int64), ("suspect_shard", C.c_void_p),
                ("suspect_index", C.c_void_p), ("suspect_missing_off", C.c_void_p),
                ("missing_capacity", C.c_int64), ("missing_ids", C.c_void_p),
                ("n_suspect", C.c_int64), ("raia_valid", C.c_int32), ("reserved1", C.c_int32)]


class CBankResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("reference_throws", C.c_int32), ("read_count", C.c_int64),
                ("error_count", C.c_int64), ("first_error_index", C.c_int32),
                ("first_error_type", C.c_int32), ("count_by_type", C.c_int64 * 5),
                ("first_index_by_type", C.c_int32 * 5), ("last_index_by_type", C.c_int32 * 5),
                ("worst_index_by_type", C.c_int32 * 5), ("lowest_total", C.c_int64),
                ("highest_total", C.c_int64), ("lowest_index", C.c_int32),
                ("highest_index", C.c_int32), ("seconds_kernel", C.c_double),
                ("seconds_total", C.c_double)]


def alloc_setfull_out(h, shards):
    """Caller-side buffers for jtb_check_set_full (returns the struct and the numpy arrays backing it)."""
    import numpy as np
    n_add_inv = int(np.count_nonzero((h.f == 3) & (h.type == 0))) + 1
    n_final = int(np.count_nonzero((h.flags & 1) != 0)) + 1
    bufs = {
        "elem_off": np.zeros(h.n_shards + 1, np.int64), "elem_id": np.zeros(n_add_inv, np.int32),
        "elem_outcome": np.zeros(n_add_inv, np.uint8), "elem_latency_ms": np.zeros(n_add_inv, np.int64),
        "elem_dup_count": np.zeros(n_add_inv, np.int32),
        "suspect_shard": np.zeros(n_final, np.int32), "suspect_index": np.zeros(n_final, np.int32),
        "suspect_missing_off": np.zeros(n_final + 1, np.int64),
        "missing_ids": np.zeros(max(1, min(n_final * n_add_inv, 1 << 26)), np.int32),
    }
    out = CSetFullOut()
    out.shards = C.cast(shards, C.c_void_p)
    out.elem_capacity = n_add_inv
    for k in ("elem_off", "elem_id", "elem_outcome", "elem_latency_ms", "elem_dup_count", "suspect_shard",
              "suspect_index", "suspect_missing_off", "missing_ids"):
        setattr(out, k, bufs[k].ctypes.data)
    out.suspect_capacity = n_final
    out.missing_capacity = bufs["missing_ids"].shape[0]
    return out, bufs


SETFULL_SHARD_FIELDS = ("valid", "attempt_count", "stable_count", "lost_count", "never_read_count", "stale_count",
                        "duplicated_count", "suspect_final_reads", "stable_latency_max_ms", "lost_latency_max_ms")


def setfull_to_dict(out, shards, bufs) -> dict:
    n = int(bufs["elem_off"][-1])
    ns = int(out.n_suspect)
    moff = bufs["suspect_missing_off"]
    return {
        "valid": out.valid, "n_failures": out.n_failures, "seconds": out.seconds_total,
        "seconds_kernel": out.seconds_kernel,
        "shards": [{f: getattr(s, f) for f in SETFULL_SHARD_FIELDS} for s in shards],
        "elem_off": bufs["elem_off"].copy(), "elem_id": bufs["elem_id"][:n].copy(),
        "elem_outcome": bufs["elem_outcome"][:n].copy(), "elem_latency_ms": bufs["elem_latency_ms"][:n].copy(),
        "elem_dup_count": bufs["elem_dup_count"][:n].copy(),
        "raia_valid": out.raia_valid,
        "suspect_final_reads": [
            {"shard": int(bufs["suspect_shard"][i]), "index": int(bufs["suspect_index"][i]),
             "missing": [int(x) for x in bufs["missing_ids"][int(moff[i]):int(moff[i + 1])]]} for i in range(ns)],
    }


class CMonoShard(C.Structure):
    """jtb_mono_shard: the monotonic-key verdict of one shard."""
    _fields_ = [("valid", C.c_int32), ("cause", C.c_int32), ("n_reads", C.c_int32), ("n_keys", C.c_int32),
                ("witness_index", C.c_int32), ("partner_index", C.c_int32), ("edge_kind", C.c_int32 * 2),
                ("edge_key", C.c_int32 * 2), ("edge_value", C.c_int64 * 2), ("edge_value2", C.c_int64 * 2)]


class CMonoResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32), ("n_reads", C.c_int64),
                ("seconds_kernel", C.c_double), ("seconds_total", C.c_double)]


MONO_SHARD_FIELDS = ("valid", "cause", "n_reads", "n_keys", "witness_index", "partner_index")


def mono_to_dict(res, shards) -> dict:
    """One result dict for the library and the oracle: edges are [partner -> witness, witness -> partner], each
    (kind, key, value, value')."""
    return {
        "valid": res.valid, "n_failures": res.n_failures, "n_reads": res.n_reads,
        "seconds_kernel": res.seconds_kernel, "seconds_total": res.seconds_total,
        "shards": [dict({f: getattr(s, f) for f in MONO_SHARD_FIELDS},
                        edges=[(s.edge_kind[i], s.edge_key[i], s.edge_value[i], s.edge_value2[i]) for i in (0, 1)])
                   for s in shards],
    }


class CCbShard(C.Structure):
    """jtb_cb_shard: the counter-bounds verdict of one shard."""
    _fields_ = [("valid", C.c_int32), ("n_reads", C.c_int32), ("n_transfers", C.c_int32), ("n_keys", C.c_int32),
                ("n_below", C.c_int64), ("n_above", C.c_int64), ("witness_index", C.c_int32),
                ("witness_key", C.c_int32), ("kind", C.c_int32), ("culprit_index", C.c_int32),
                ("value", C.c_int64), ("bound", C.c_int64)]


class CCbResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32), ("n_reads", C.c_int64), ("n_transfers", C.c_int64),
                ("n_violations", C.c_int64), ("seconds_kernel", C.c_double), ("seconds_total", C.c_double)]


CB_SHARD_FIELDS = ("valid", "n_reads", "n_transfers", "n_keys", "n_below", "n_above", "witness_index", "witness_key",
                   "kind", "culprit_index", "value", "bound")


def cb_to_dict(res, shards) -> dict:
    """One result dict for the library and the oracle."""
    return {
        "valid": res.valid, "n_failures": res.n_failures, "n_reads": res.n_reads, "n_transfers": res.n_transfers,
        "n_violations": res.n_violations, "seconds_kernel": res.seconds_kernel, "seconds_total": res.seconds_total,
        "shards": [{f: getattr(s, f) for f in CB_SHARD_FIELDS} for s in shards],
    }


class CTlShard(C.Structure):
    """jtb_tl_shard: the transfer-lookup verdict of one shard."""
    _fields_ = [("valid", C.c_int32), ("n_lookups", C.c_int32), ("n_records", C.c_int64), ("n_transfers", C.c_int32),
                ("n_reads", C.c_int32), ("count_by_kind", C.c_int64 * TL_KINDS), ("witness_index", C.c_int32),
                ("kind", C.c_int32), ("transfer_id", C.c_int64), ("key", C.c_int32), ("related_index", C.c_int32),
                ("value", C.c_int64), ("bound", C.c_int64)]


class CTlResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32), ("n_lookups", C.c_int64), ("n_records", C.c_int64),
                ("n_transfers", C.c_int64), ("n_reads", C.c_int64), ("n_violations", C.c_int64),
                ("seconds_kernel", C.c_double), ("seconds_total", C.c_double)]


TL_SHARD_FIELDS = ("valid", "n_lookups", "n_records", "n_transfers", "n_reads", "count_by_kind", "witness_index",
                   "kind", "transfer_id", "key", "related_index", "value", "bound")


def tl_to_dict(res, shards) -> dict:
    """One result dict for the library and the oracle (count_by_kind as a list indexed by kind - 1)."""
    return {
        "valid": res.valid, "n_failures": res.n_failures, "n_lookups": res.n_lookups, "n_records": res.n_records,
        "n_transfers": res.n_transfers, "n_reads": res.n_reads, "n_violations": res.n_violations,
        "seconds_kernel": res.seconds_kernel, "seconds_total": res.seconds_total,
        "shards": [{f: (list(s.count_by_kind) if f == "count_by_kind" else getattr(s, f)) for f in TL_SHARD_FIELDS}
                   for s in shards],
    }


class CRxShard(C.Structure):
    """jtb_rx_shard: the read-explanation verdict of one shard."""
    _fields_ = [("valid", C.c_int32), ("n_reads", C.c_int32), ("n_transfers", C.c_int32), ("witness_index", C.c_int32),
                ("n_explained", C.c_int64), ("n_undecided", C.c_int64), ("count_by_kind", C.c_int64 * 2),
                ("nodes", C.c_int64), ("kind", C.c_int32), ("key", C.c_int32), ("n_must", C.c_int32),
                ("n_may", C.c_int32), ("value", C.c_int64), ("must_sum", C.c_int64)]


class CRxResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32), ("n_reads", C.c_int64), ("n_transfers", C.c_int64),
                ("n_explained", C.c_int64), ("n_unexplained", C.c_int64), ("n_undecided", C.c_int64),
                ("nodes", C.c_int64), ("seconds_kernel", C.c_double), ("seconds_total", C.c_double)]


RX_SHARD_FIELDS = ("valid", "n_reads", "n_transfers", "witness_index", "n_explained", "n_undecided", "count_by_kind",
                   "nodes", "kind", "key", "n_must", "n_may", "value", "must_sum")


def rx_to_dict(res, shards) -> dict:
    """One result dict for the library and the oracle (count_by_kind as a list indexed by kind - 1)."""
    return {
        "valid": res.valid, "n_failures": res.n_failures, "n_reads": res.n_reads, "n_transfers": res.n_transfers,
        "n_explained": res.n_explained, "n_unexplained": res.n_unexplained, "n_undecided": res.n_undecided,
        "nodes": res.nodes, "seconds_kernel": res.seconds_kernel, "seconds_total": res.seconds_total,
        "shards": [{f: (list(s.count_by_kind) if f == "count_by_kind" else getattr(s, f)) for f in RX_SHARD_FIELDS}
                   for s in shards],
    }


class CRgShard(C.Structure):
    """jtb_rg_shard: the read-gap verdict of one shard."""
    _fields_ = [("valid", C.c_int32), ("cause", C.c_int32), ("n_reads", C.c_int32), ("n_transfers", C.c_int32),
                ("n_explained", C.c_int64), ("n_undecided", C.c_int64), ("count_by_kind", C.c_int64 * 3),
                ("nodes", C.c_int64), ("witness_index", C.c_int32), ("lower_index", C.c_int32), ("kind", C.c_int32),
                ("key", C.c_int32), ("delta", C.c_int64), ("transfer_id", C.c_int64), ("other_index", C.c_int32),
                ("n_eligible", C.c_int32)]


class CRgResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32), ("n_reads", C.c_int64), ("n_transfers", C.c_int64),
                ("n_explained", C.c_int64), ("n_unexplained", C.c_int64), ("n_double", C.c_int64),
                ("n_undecided", C.c_int64), ("nodes", C.c_int64), ("seconds_kernel", C.c_double),
                ("seconds_total", C.c_double)]


RG_SHARD_FIELDS = ("valid", "cause", "n_reads", "n_transfers", "n_explained", "n_undecided", "count_by_kind", "nodes",
                   "witness_index", "lower_index", "kind", "key", "delta", "transfer_id", "other_index", "n_eligible")


def rg_to_dict(res, shards) -> dict:
    """One result dict for the library and the oracle (count_by_kind as a list indexed by kind - 1)."""
    return {
        "valid": res.valid, "n_failures": res.n_failures, "n_reads": res.n_reads, "n_transfers": res.n_transfers,
        "n_explained": res.n_explained, "n_unexplained": res.n_unexplained, "n_double": res.n_double,
        "n_undecided": res.n_undecided, "nodes": res.nodes, "seconds_kernel": res.seconds_kernel,
        "seconds_total": res.seconds_total,
        "shards": [{f: (list(s.count_by_kind) if f == "count_by_kind" else getattr(s, f)) for f in RG_SHARD_FIELDS}
                   for s in shards],
    }


class CTpShard(C.Structure):
    """jtb_tp_shard: the transfer-placement verdict of one shard."""
    _fields_ = [("valid", C.c_int32), ("cause", C.c_int32), ("n_reads", C.c_int32), ("n_transfers", C.c_int32),
                ("n_explained", C.c_int64), ("n_undecided", C.c_int64), ("count_by_kind", C.c_int64 * 4),
                ("n_placed", C.c_int64), ("nodes", C.c_int64), ("rounds", C.c_int32), ("witness_index", C.c_int32),
                ("lower_index", C.c_int32), ("kind", C.c_int32), ("key", C.c_int32), ("round", C.c_int32),
                ("delta", C.c_int64), ("transfer_id", C.c_int64), ("other_index", C.c_int32),
                ("n_eligible", C.c_int32)]


class CTpResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32), ("n_reads", C.c_int64), ("n_transfers", C.c_int64),
                ("n_explained", C.c_int64), ("n_unexplained", C.c_int64), ("n_double", C.c_int64),
                ("n_lost", C.c_int64), ("n_undecided", C.c_int64), ("n_placed", C.c_int64), ("nodes", C.c_int64),
                ("rounds", C.c_int64), ("seconds_kernel", C.c_double), ("seconds_total", C.c_double)]


TP_SHARD_FIELDS = ("valid", "cause", "n_reads", "n_transfers", "n_explained", "n_undecided", "count_by_kind",
                   "n_placed", "nodes", "rounds", "witness_index", "lower_index", "kind", "key", "round", "delta",
                   "transfer_id", "other_index", "n_eligible")


def tp_to_dict(res, shards) -> dict:
    """One result dict for the library and the oracle (count_by_kind as a list indexed by kind - 1)."""
    return {
        "valid": res.valid, "n_failures": res.n_failures, "n_reads": res.n_reads, "n_transfers": res.n_transfers,
        "n_explained": res.n_explained, "n_unexplained": res.n_unexplained, "n_double": res.n_double,
        "n_lost": res.n_lost, "n_undecided": res.n_undecided, "n_placed": res.n_placed, "nodes": res.nodes,
        "rounds": res.rounds, "seconds_kernel": res.seconds_kernel, "seconds_total": res.seconds_total,
        "shards": [{f: (list(s.count_by_kind) if f == "count_by_kind" else getattr(s, f)) for f in TP_SHARD_FIELDS}
                   for s in shards],
    }


class CSwShard(C.Structure):
    """jtb_sw_shard: the serial-witness verdict of one shard."""
    _fields_ = [("valid", C.c_int32), ("cause", C.c_int32), ("n_reads", C.c_int32), ("n_transfers", C.c_int32),
                ("n_committed", C.c_int64), ("n_committed_crashed", C.c_int64), ("n_after", C.c_int64),
                ("nodes", C.c_int64), ("rounds", C.c_int32), ("fail_index", C.c_int32), ("transfer_id", C.c_int64)]


class CSwResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("n_failures", C.c_int32), ("n_reads", C.c_int64), ("n_transfers", C.c_int64),
                ("n_committed", C.c_int64), ("n_committed_crashed", C.c_int64), ("n_after", C.c_int64),
                ("nodes", C.c_int64), ("rounds", C.c_int64), ("seconds_kernel", C.c_double),
                ("seconds_total", C.c_double)]


def _names(struct) -> tuple:
    return tuple(f for f, _ in struct._fields_)


SW_SHARD_FIELDS = _names(CSwShard)
SW_RESULT_FIELDS = _names(CSwResult)


def witness_to_dict(res, shards, commit_read=None, lookup_read=None) -> dict:
    """One result dict of a witness check (jtb_sw_* .. jtb_lk_*, K13-K17) for the library and the oracle: the
    result's fields and "shards" with each shard's; "commit_read" (a numpy int32 array, one entry per transfer micro-op
    in history order) and "lookup_read" (one entry per :ok lookup in history order) when they were asked for."""
    out = {f: getattr(res, f) for f, _ in res._fields_}
    out["shards"] = [{f: getattr(s, f) for f, _ in s._fields_} for s in shards]
    if commit_read is not None:
        out["commit_read"] = commit_read
    if lookup_read is not None:
        out["lookup_read"] = lookup_read
    return out


RW_DEFAULT_MAX_REPAIRS = 32


class CRwShard(C.Structure):
    """jtb_rw_shard: the repaired-serial-witness verdict of one shard."""
    _fields_ = CSwShard._fields_ + [("repairs", C.c_int32), ("n_bans", C.c_int32)]


class CRwResult(C.Structure):
    _fields_ = CSwResult._fields_[:9] + [("repairs", C.c_int64), ("n_bans", C.c_int64)] + CSwResult._fields_[9:]


RW_SHARD_FIELDS = _names(CRwShard)
RW_RESULT_FIELDS = _names(CRwResult)


LW_DEFAULT_MAX_LIFTS = 32


class CLwShard(C.Structure):
    """jtb_lw_shard: the lifted-serial-witness verdict of one shard."""
    _fields_ = CRwShard._fields_ + [("lifts", C.c_int32), ("n_lifted", C.c_int32)]


class CLwResult(C.Structure):
    _fields_ = CRwResult._fields_[:11] + [("lifts", C.c_int64), ("n_lifted", C.c_int64)] + CRwResult._fields_[11:]


LW_SHARD_FIELDS = _names(CLwShard)
LW_RESULT_FIELDS = _names(CLwResult)


class CCwShard(C.Structure):
    """jtb_cw_shard: the class-witness verdict of one shard."""
    _fields_ = CLwShard._fields_ + [("class_cause", C.c_int32), ("class_rounds", C.c_int32), ("n_handed", C.c_int64)]


class CCwResult(C.Structure):
    _fields_ = CLwResult._fields_[:13] + [("class_rounds", C.c_int64), ("n_handed", C.c_int64)] + \
        CLwResult._fields_[13:]


CW_SHARD_FIELDS = _names(CCwShard)
CW_RESULT_FIELDS = _names(CCwResult)


class CLkShard(C.Structure):
    """jtb_lk_shard: the lookup-witness verdict of one shard."""
    _fields_ = CCwShard._fields_ + [("lookup_cause", C.c_int32), ("lookup_fail_index", C.c_int32),
                                    ("n_lookups_placed", C.c_int64)]


class CLkResult(C.Structure):
    _fields_ = CCwResult._fields_[:15] + [("n_lookups_placed", C.c_int64)] + CCwResult._fields_[15:]


CAUSE_LOOKUP = 9
LK_SHARD_FIELDS = _names(CLkShard)
LK_RESULT_FIELDS = _names(CLkResult)


def n_ok_lookups(h) -> int:
    """:ok lookups of a ledger-lookups history."""
    import numpy as np
    return int(np.sum((h.type == 1) & (h.f == 5) & (h.process >= 0) & (h.payload_len >= 0)))


def n_transfer_records(h) -> int:
    """Transfer micro-ops of a ledger-lookups history: the records of its transfer invokes."""
    import numpy as np
    inv = (h.type == 0) & (h.f == 4) & (h.process >= 0) & (h.payload_len > 0)
    return int(np.sum(h.payload_len[inv] // 5))


# ---- K18: the stored-history reader --------------------------------------------------------------------------------
FORM_BANK, FORM_LEDGER_COUNTERS, FORM_LEDGER_LOOKUPS = 0, 1, 2
FORMS = {"bank": FORM_BANK, "ledger-counters": FORM_LEDGER_COUNTERS, "ledger-lookups": FORM_LEDGER_LOOKUPS}


class CEdnHistory(C.Structure):
    """ctypes image of `struct jtb_edn_history`."""

    _fields_ = [("history", CHistory), ("multi_transfer_txns", C.c_int64), ("n_ops", C.c_int64),
                ("seconds_h2d", C.c_double), ("seconds_kernel", C.c_double), ("seconds_d2h", C.c_double),
                ("seconds_total", C.c_double)]


# ---- K19: the host checks of a ledger compose on a stored history.edn ----------------------------------------------
class CEdnFlag(C.Structure):
    """ctypes image of `struct jtb_edn_flag`: one flagged op of a stored history."""

    _fields_ = [("op", C.c_int64), ("begin", C.c_int64), ("end", C.c_int64), ("time", C.c_int64),
                ("first", C.c_int64), ("index", C.c_int32), ("cls", C.c_int32), ("has_time", C.c_uint8),
                ("has_index", C.c_uint8), ("suspect", C.c_uint8), ("pad", C.c_uint8 * 5)]


EDN_FLAG_DTYPE = [("op", "<i8"), ("begin", "<i8"), ("end", "<i8"), ("time", "<i8"), ("first", "<i8"),
                  ("index", "<i4"), ("cls", "<i4"), ("has_time", "u1"), ("has_index", "u1"), ("suspect", "u1"),
                  ("pad", "u1", (5,))]
EDN_CHECKS_COUNTS = ("n_ops", "n_client", "n_ok", "n_fail", "n_info", "n_open", "n_final_reads", "n_final_lookups",
                     "n_read_classes", "n_lookup_classes", "n_invoked", "n_suspect")


class CEdnChecks(C.Structure):
    """ctypes image of `struct jtb_edn_checks`."""

    _fields_ = ([(name, C.c_int64) for name in EDN_CHECKS_COUNTS]
                + [("last", CEdnFlag), ("open", C.c_void_p), ("fails", C.c_void_p), ("final_reads", C.c_void_p),
                   ("final_lookups", C.c_void_p), ("refused", C.c_int32), ("reserved", C.c_int32),
                   ("refused_at", C.c_int64), ("refused_reason", C.c_char * 128), ("seconds_h2d", C.c_double),
                   ("seconds_kernel", C.c_double), ("seconds_d2h", C.c_double), ("seconds_total", C.c_double)])
