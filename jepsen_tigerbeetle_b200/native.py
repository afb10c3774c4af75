"""ctypes binding of the product library `libjtb_check.so` (C ABI in include/jtb_check.h).

This is the same boundary a JVM host binds through JNI (see INTEGRATION.md).  There is NO fallback:
if the CUDA library is missing or no device is present, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

from . import abi
from .history import CModel, FlatHistory, as_c_history

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("JTB_LIB_PATH") or os.path.join(_HERE, "libjtb_check.so")  # env: A/B experiments only
CSRC = os.path.join(_HERE, "csrc")
_SOURCES = ["jtb_abi.cu", "jtb_prep.cpp", "jtb_multi.cpp"]
_DEPS = _SOURCES + ["jtb_prep.h", "jtb_expand.h", "jtb_wgl.cuh", "jtb_scout.cuh", "jtb_scans.cuh",
                    "jtb_table_bench.cuh", "jtb_level.cuh", "jtb_partition.cuh", "jtb_monotonic.cuh",
                    "jtb_counter_bounds.cuh", "jtb_transfer_lookups.cuh", "jtb_read_explanations.cuh",
                    "jtb_read_gaps.cuh", "jtb_transfer_placement.cuh", "jtb_serial_witness.cuh", "jtb_repaired_witness.cuh",
                    "jtb_lifted_witness.cuh", "jtb_class_witness.cuh", "jtb_lookup_witness.cuh", "jtb_call.cuh"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared", "-ldl"]

EXPORTS = ["jtb_abi_version", "jtb_device_count", "jtb_create", "jtb_destroy", "jtb_last_error",
           "jtb_check_linearizable", "jtb_check_set_full", "jtb_check_bank_totals", "jtb_check_monotonic_keys",
           "jtb_check_counter_bounds", "jtb_check_transfer_lookups", "jtb_check_read_explanations",
           "jtb_check_read_gaps", "jtb_check_transfer_placement", "jtb_check_serial_witness",
           "jtb_check_repaired_witness", "jtb_check_lifted_witness", "jtb_check_class_witness",
           "jtb_check_lookup_witness",
           "jtb_table_bench", "jtb_get_stats", "jtb_struct_size", "jtb_prepare_seconds", "jtb_prepare_info",
           "jtb_final_configs", "jtb_gather_bench", "jtb_host_alloc", "jtb_host_free", "jtb_partition_by_key", "jtb_ledger_balances", "jtb_multi_create", "jtb_multi_create_error", "jtb_multi_destroy", "jtb_multi_n_gpus",
           "jtb_multi_last_error", "jtb_multi_check_linearizable", "jtb_multi_check_set_full"]

_lib = None
_lock = threading.Lock()


class NativeError(RuntimeError):
    pass


def build(force: bool = False) -> str:
    """Compile the CUDA library in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    deps = [os.path.join(CSRC, f) for f in _DEPS]
    deps.append(os.path.join(_HERE, "..", "include", "jtb_check.h"))
    stale = (not os.path.exists(LIB_PATH)
             or any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in deps))
    if force or stale:
        cmd = ["nvcc", *NVCC_FLAGS, "-o", LIB_PATH] + [os.path.join(CSRC, f) for f in _SOURCES]
        subprocess.check_call(cmd)
    return LIB_PATH


def lib() -> C.CDLL:
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise NativeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; "
                                  "g.build()'` (there is no CPU fallback)")
            L = C.CDLL(LIB_PATH)
            L.jtb_abi_version.restype = C.c_int
            L.jtb_struct_size.restype = C.c_long
            L.jtb_prepare_seconds.restype = C.c_double
            L.jtb_prepare_seconds.argtypes = [C.c_void_p, C.c_void_p]
            L.jtb_prepare_info.restype = C.c_double
            L.jtb_prepare_info.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
            L.jtb_device_count.restype = C.c_int
            L.jtb_create.restype = C.c_void_p
            L.jtb_create.argtypes = [C.c_void_p]
            L.jtb_destroy.argtypes = [C.c_void_p]
            L.jtb_last_error.restype = C.c_char_p
            L.jtb_last_error.argtypes = [C.c_void_p]
            L.jtb_check_linearizable.argtypes = [C.c_void_p] * 5
            L.jtb_final_configs.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
            L.jtb_check_set_full.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
            L.jtb_check_bank_totals.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
            L.jtb_check_monotonic_keys.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
            L.jtb_check_counter_bounds.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
            L.jtb_check_transfer_lookups.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
            L.jtb_check_read_explanations.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                                      C.c_void_p]
            L.jtb_check_read_gaps.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
            L.jtb_check_transfer_placement.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                                       C.c_void_p, C.c_void_p]
            L.jtb_check_serial_witness.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]
            L.jtb_check_repaired_witness.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                                     C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
            L.jtb_check_lifted_witness.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                                   C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
            L.jtb_check_class_witness.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                                  C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
            L.jtb_check_lookup_witness.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32,
                                                   C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]
            L.jtb_table_bench.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_void_p,
                                          C.c_void_p, C.c_void_p]
            L.jtb_gather_bench.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_uint32, C.c_int, C.c_int,
                                           C.c_void_p, C.c_void_p]
            L.jtb_multi_create.restype = C.c_void_p
            L.jtb_multi_create.argtypes = [C.c_void_p, C.c_int]
            L.jtb_multi_create_error.restype = C.c_char_p
            L.jtb_multi_destroy.argtypes = [C.c_void_p]
            L.jtb_multi_n_gpus.argtypes = [C.c_void_p]
            L.jtb_multi_last_error.restype = C.c_char_p
            L.jtb_multi_last_error.argtypes = [C.c_void_p]
            L.jtb_multi_check_linearizable.argtypes = [C.c_void_p] * 6
            L.jtb_multi_check_set_full.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
            if L.jtb_abi_version() != abi.ABI_VERSION:
                raise NativeError("ABI version mismatch between libjtb_check.so and abi.py")
            _lib = L
    return _lib


class Context:
    """One checker context = one CUDA device + stream + cached device buffers (`jtb_ctx`)."""

    def __init__(self, device: int = 0, table_bytes: int = 0, max_configs: int = 0,
                 time_budget_ms: int = 0, search_ctas: int = 0, eager_reads: bool = True,
                 scouts: bool = True, engine: str = "auto", beam: bool = True) -> None:
        """engine: "auto" (chosen from the history, DESIGN.md section 4), "level", "worklist"; beam=False skips the beam
        sweep that histories with crashed ops get first."""
        L = lib()
        flags = (0 if eager_reads else abi.OPT_NO_EAGER_READS) | (0 if scouts else abi.OPT_NO_SCOUTS)
        flags |= {"auto": 0, "level": abi.OPT_ENGINE_LEVEL, "worklist": abi.OPT_ENGINE_WORKLIST}[engine]
        flags |= 0 if beam else abi.OPT_NO_BEAM
        opts = abi.COpts(device, flags, table_bytes, max_configs, time_budget_ms, search_ctas)
        self._h = L.jtb_create(C.byref(opts))
        if not self._h:
            raise NativeError("jtb_create failed: no CUDA device available (no CPU fallback)")

    def close(self) -> None:
        if getattr(self, "_h", None):
            lib().jtb_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _err(self) -> str:
        return lib().jtb_last_error(self._h).decode()

    # ---- hot path A9 ----------------------------------------------------------------------------
    def check_linearizable(self, h: FlatHistory, model: CModel) -> dict:
        ch = as_c_history(h)
        shards = (abi.CLinShard * h.n_shards)()
        res = abi.CLinResult()
        rc = lib().jtb_check_linearizable(self._h, C.addressof(ch), C.addressof(model),
                                          C.addressof(shards), C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_linearizable rc={rc}: {self._err()}")
        return {
            "valid": res.valid, "n_failures": res.n_failures, "configs": res.configs_explored,
            "probes": res.probes, "hbm_bytes_algorithmic": res.hbm_bytes_algorithmic,
            "key_bytes": res.key_bytes, "seconds_kernel": res.seconds_kernel,
            "seconds_total": res.seconds_total,
            "shards": [{"valid": s.valid, "witness_index": s.witness_index,
                        "previous_ok_index": s.previous_ok_index, "cause": s.cause,
                        "configs": s.configs_explored, "probes": s.probes} for s in shards],
        }

    # ---- hot path A4 ----------------------------------------------------------------------------
    def check_set_full(self, h: FlatHistory, linearizable: bool = True) -> dict:
        ch = as_c_history(h)
        shards = (abi.CSetFullShard * h.n_shards)()
        out, bufs = abi.alloc_setfull_out(h, shards)
        rc = lib().jtb_check_set_full(self._h, C.addressof(ch), int(linearizable), C.addressof(out))
        if rc != 0:
            raise NativeError(f"jtb_check_set_full rc={rc}: {self._err()}")
        return abi.setfull_to_dict(out, shards, bufs)

    # ---- hot path A8 ----------------------------------------------------------------------------
    def check_bank_totals(self, h: FlatHistory, model: CModel, total_amount: int = 0) -> dict:
        ch = as_c_history(h)
        res = abi.CBankResult()
        rc = lib().jtb_check_bank_totals(self._h, C.addressof(ch), C.addressof(model),
                                         C.c_int64(total_amount), C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_bank_totals rc={rc}: {self._err()}")
        return {
            "valid": res.valid, "reference_throws": res.reference_throws, "read_count": res.read_count,
            "error_count": res.error_count,
            "first_error_index": res.first_error_index, "first_error_type": res.first_error_type,
            "count_by_type": list(res.count_by_type),
            "first_index_by_type": list(res.first_index_by_type),
            "last_index_by_type": list(res.last_index_by_type),
            "worst_index_by_type": list(res.worst_index_by_type),
            "lowest_total": res.lowest_total, "highest_total": res.highest_total,
            "lowest_index": res.lowest_index, "highest_index": res.highest_index,
            "seconds": res.seconds_total, "seconds_kernel": res.seconds_kernel,
        }

    # ---- K7: monotonic-key check ------------------------------------------------------------------
    def check_monotonic_keys(self, h: FlatHistory, realtime: bool = True) -> dict:
        """Elle's monotonic-key graph (plus real-time order unless realtime=False) over the :ok reads of every shard:
        {"valid", "n_failures", "n_reads", "seconds_kernel", "seconds_total", "shards": [{"valid", "cause", "n_reads",
        "n_keys", "witness_index", "partner_index", "edges": [(kind, key, value, value') partner->witness,
        witness->partner]}]}.  Read payloads are (key, value_lo, value_hi) triples (flatten_ops(..., "ledger-counters"))."""
        ch = as_c_history(h)
        shards = (abi.CMonoShard * max(1, h.n_shards))()
        res = abi.CMonoResult()
        rc = lib().jtb_check_monotonic_keys(self._h, C.addressof(ch), 0 if realtime else abi.MONO_NO_REALTIME,
                                            C.addressof(shards), C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_monotonic_keys rc={rc}: {self._err()}")
        return abi.mono_to_dict(res, shards[:h.n_shards])

    # ---- K8: counter-bounds check -----------------------------------------------------------------
    def check_counter_bounds(self, h: FlatHistory) -> dict:
        """Every counter an :ok read observes against the transfers around it: L (the :ok transfers completed before
        the read was invoked) <= value <= U (the non-:fail transfers invoked before it completed).
        {"valid", "n_failures", "n_reads", "n_transfers", "n_violations", "seconds_kernel", "seconds_total",
        "shards": [{"valid", "n_reads", "n_transfers", "n_keys", "n_below", "n_above", "witness_index", "witness_key",
        "kind", "culprit_index", "value", "bound"}]}.  Input as for check_monotonic_keys."""
        ch = as_c_history(h)
        shards = (abi.CCbShard * max(1, h.n_shards))()
        res = abi.CCbResult()
        rc = lib().jtb_check_counter_bounds(self._h, C.addressof(ch), 0, C.addressof(shards), C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_counter_bounds rc={rc}: {self._err()}")
        return abi.cb_to_dict(res, shards[:h.n_shards])

    # ---- K9: transfer-lookup check ------------------------------------------------------------------
    def check_transfer_lookups(self, h: FlatHistory) -> dict:
        """The transfer records :ok lookups return against the transfers clients issued and the counters reads show
        (input: the ledger-lookups form).  {"valid", "n_failures", "n_lookups", "n_records", "n_transfers", "n_reads",
        "n_violations", "seconds_kernel", "seconds_total", "shards": [{"valid", "n_lookups", "n_records",
        "n_transfers", "n_reads", "count_by_kind", "witness_index", "kind", "transfer_id", "key", "related_index",
        "value", "bound"}]}; count_by_kind[kind - 1]."""
        ch = as_c_history(h)
        shards = (abi.CTlShard * max(1, h.n_shards))()
        res = abi.CTlResult()
        rc = lib().jtb_check_transfer_lookups(self._h, C.addressof(ch), 0, C.addressof(shards), C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_transfer_lookups rc={rc}: {self._err()}")
        return abi.tl_to_dict(res, shards[:h.n_shards])

    # ---- K10: read-explanation check ----------------------------------------------------------------
    def check_read_explanations(self, h: FlatHistory, max_nodes: int = 0) -> dict:
        """Does one set of transfers explain every counter each :ok read shows?  The transfers that must be in the read,
        the ones that cannot be and the ones that may be, and a budgeted subset-sum search over the last (input: the
        ledger-lookups form; max_nodes <= 0 is the default budget).  {"valid", "n_failures", "n_reads", "n_transfers",
        "n_explained", "n_unexplained", "n_undecided", "nodes", "seconds_kernel", "seconds_total", "shards": [{"valid",
        "n_reads", "n_transfers", "witness_index", "n_explained", "n_undecided", "count_by_kind", "nodes", "kind",
        "key", "n_must", "n_may", "value", "must_sum"}]}; count_by_kind[kind - 1]."""
        ch = as_c_history(h)
        shards = (abi.CRxShard * max(1, h.n_shards))()
        res = abi.CRxResult()
        rc = lib().jtb_check_read_explanations(self._h, C.addressof(ch), max_nodes, 0, C.addressof(shards),
                                               C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_read_explanations rc={rc}: {self._err()}")
        return abi.rx_to_dict(res, shards[:h.n_shards])

    # ---- K11: read-gap check ------------------------------------------------------------------------------------
    def check_read_gaps(self, h: FlatHistory, max_nodes: int = 0) -> dict:
        """Do the transfers committed between two successive :ok reads (in the monotonic-key order) explain what
        changed?  A budgeted subset-sum search per gap over the transfers eligible for it, and no transfer forced into
        two gaps (input: the ledger-lookups form; max_nodes <= 0 is the default budget).  {"valid", "n_failures",
        "n_reads", "n_transfers", "n_explained", "n_unexplained", "n_double", "n_undecided", "nodes", "seconds_kernel",
        "seconds_total", "shards": [{"valid", "cause", "n_reads", "n_transfers", "n_explained", "n_undecided",
        "count_by_kind", "nodes", "witness_index", "lower_index", "kind", "key", "delta", "transfer_id",
        "other_index", "n_eligible"}]}; count_by_kind[kind - 1]."""
        ch = as_c_history(h)
        shards = (abi.CRgShard * max(1, h.n_shards))()
        res = abi.CRgResult()
        rc = lib().jtb_check_read_gaps(self._h, C.addressof(ch), max_nodes, 0, C.addressof(shards), C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_read_gaps rc={rc}: {self._err()}")
        return abi.rg_to_dict(res, shards[:h.n_shards])

    # ---- K12: transfer-placement check ---------------------------------------------------------------------------
    def check_transfer_placement(self, h: FlatHistory, max_nodes: int = 0, max_rounds: int = 0) -> dict:
        """The read-gap check, with every transfer a gap's root pruning locates (or that only one gap of its window
        can still hold) carried into the other gaps, round after round to a fixpoint; a transfer known to be committed
        that no gap of its window can hold is LOST (input: the ledger-lookups form; max_nodes <= 0 and max_rounds <= 0
        are the defaults).  {"valid", "n_failures", "n_reads", "n_transfers", "n_explained", "n_unexplained",
        "n_double", "n_lost", "n_undecided", "n_placed", "nodes", "rounds", "seconds_kernel", "seconds_total",
        "shards": [{"valid", "cause", "n_reads", "n_transfers", "n_explained", "n_undecided", "count_by_kind",
        "n_placed", "nodes", "rounds", "witness_index", "lower_index", "kind", "key", "round", "delta", "transfer_id",
        "other_index", "n_eligible"}]}; count_by_kind[kind - 1]."""
        ch = as_c_history(h)
        shards = (abi.CTpShard * max(1, h.n_shards))()
        res = abi.CTpResult()
        rc = lib().jtb_check_transfer_placement(self._h, C.addressof(ch), max_nodes, max_rounds, 0,
                                                C.addressof(shards), C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_transfer_placement rc={rc}: {self._err()}")
        return abi.tp_to_dict(res, shards[:h.n_shards])

    # ---- K13: serial-witness check --------------------------------------------------------------------------------
    def check_serial_witness(self, h: FlatHistory, max_nodes: int = 0, max_rounds: int = 0,
                             witness: bool = False) -> dict:
        """A proof of linearizability, or nothing: the transfer-placement check, then one explanation chosen per read
        gap (no transfer in two) and the serial order it gives checked against real time.  A shard is VALID (its reads
        and transfers are linearizable for the per-account counters, and so for the bank model with negative balances
        allowed) or UNKNOWN with a cause, never INVALID (input: the ledger-lookups form; max_nodes and max_rounds as for
        check_transfer_placement).  {"valid", "n_failures", "n_reads", "n_transfers", "n_committed",
        "n_committed_crashed", "n_after", "nodes", "rounds", "seconds_kernel", "seconds_total", "shards": [{"valid",
        "cause", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes", "rounds",
        "fail_index", "transfer_id"}]}; witness=True adds "commit_read": per transfer micro-op in history order, the
        completion :index of the first read whose state holds it, abi.SW_NEVER, SW_AFTER or SW_FREE."""
        import numpy as np
        ch = as_c_history(h)
        shards = (abi.CSwShard * max(1, h.n_shards))()
        res = abi.CSwResult()
        cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32) if witness else None
        rc = lib().jtb_check_serial_witness(self._h, C.addressof(ch), max_nodes, max_rounds, 0,
                                            cr.ctypes.data if witness else None, C.addressof(shards),
                                            C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_serial_witness rc={rc}: {self._err()}")
        return abi.sw_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)

    # ---- K14: repaired serial witness ----------------------------------------------------------------------------
    def check_repaired_witness(self, h: FlatHistory, max_nodes: int = 0, max_rounds: int = 0, max_repairs: int = 0,
                               witness: bool = False, flags: int = 0) -> dict:
        """check_serial_witness, then up to max_repairs repair rounds (<= 0: abi.RW_DEFAULT_MAX_REPAIRS) on a shard it
        leaves no-witness or real-time: the failure's (transfer, gap) pairs are banned, their gaps released and the
        witness rounds run again; every VALID is the same proof.  A shard check_serial_witness proves comes back as it
        returns it.  The dict of check_serial_witness with "repairs" (the most of any shard) and "n_bans" added, and
        per shard "repairs" and "n_bans"; flags must be 0."""
        import numpy as np
        ch = as_c_history(h)
        shards = (abi.CRwShard * max(1, h.n_shards))()
        res = abi.CRwResult()
        cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32) if witness else None
        rc = lib().jtb_check_repaired_witness(self._h, C.addressof(ch), max_nodes, max_rounds, max_repairs, flags,
                                              cr.ctypes.data if witness else None, C.addressof(shards),
                                              C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_repaired_witness rc={rc}: {self._err()}")
        return abi.rw_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)

    # ---- K15: lifted serial witness ------------------------------------------------------------------------------
    def check_lifted_witness(self, h: FlatHistory, max_nodes: int = 0, max_rounds: int = 0, max_repairs: int = 0,
                             max_lifts: int = 0, witness: bool = False, flags: int = 0) -> dict:
        """check_repaired_witness, then, on a shard whose repairs stopped because a repair recorded no new ban, up to
        max_lifts lift steps (<= 0: abi.LW_DEFAULT_MAX_LIFTS): the failing gaps steal again with their own bans
        ignored, a kept thief's bans on its loot are lifted (once per pair) and the repairs resume; every VALID is the
        same proof.  A shard check_repaired_witness proves comes back as it returns it.  The dict of
        check_repaired_witness with "lifts" (the most of any shard) and "n_lifted" added, and per shard "lifts" and
        "n_lifted"; flags must be 0."""
        import numpy as np
        ch = as_c_history(h)
        shards = (abi.CLwShard * max(1, h.n_shards))()
        res = abi.CLwResult()
        cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32) if witness else None
        rc = lib().jtb_check_lifted_witness(self._h, C.addressof(ch), max_nodes, max_rounds, max_repairs, max_lifts,
                                            flags, cr.ctypes.data if witness else None, C.addressof(shards),
                                            C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_lifted_witness rc={rc}: {self._err()}")
        return abi.lw_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)

    # ---- K16: class witness --------------------------------------------------------------------------------------
    def check_class_witness(self, h: FlatHistory, max_nodes: int = 0, max_rounds: int = 0, max_repairs: int = 0,
                            max_lifts: int = 0, witness: bool = False, flags: int = 0) -> dict:
        """check_lifted_witness, then a class pass on every shard it leaves UNKNOWN (undecided, no-witness or
        real-time): from the transfer-placement check's owners, witness rounds that take at most cap members of each
        class of interchangeable crashed transfers and hand the members out earliest first, checked by the same
        real-time pass and re-sum.  A shard check_lifted_witness proves comes back as it returns it.  The dict of
        check_lifted_witness with "class_rounds" (the most of any shard) and "n_handed" added, and per shard
        "class_cause", "class_rounds" and "n_handed"; flags must be 0."""
        import numpy as np
        ch = as_c_history(h)
        shards = (abi.CCwShard * max(1, h.n_shards))()
        res = abi.CCwResult()
        cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32) if witness else None
        rc = lib().jtb_check_class_witness(self._h, C.addressof(ch), max_nodes, max_rounds, max_repairs, max_lifts,
                                           flags, cr.ctypes.data if witness else None, C.addressof(shards),
                                           C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_class_witness rc={rc}: {self._err()}")
        return abi.cw_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)

    # ---- K17: lookup witness -------------------------------------------------------------------------------------
    def check_lookup_witness(self, h: FlatHistory, max_nodes: int = 0, max_rounds: int = 0, max_repairs: int = 0,
                             max_lifts: int = 0, witness: bool = False, flags: int = 0) -> dict:
        """check_class_witness, then every :ok lookup of a shard it proves is placed in the shard's serial order: each
        lookup at a point where it returns exactly the transfers committed before it, the lookups of one read gap
        nested, and one real-time pass over the reads, transfers and lookups together.  A shard whose lookups cannot
        be placed is UNKNOWN with cause "lookup".  The dict of check_class_witness with "n_lookups_placed" added, and
        per shard "lookup_cause", "lookup_fail_index" and "n_lookups_placed"; with witness=True also "lookup_read" (one
        entry per :ok lookup in history order).  flags must be 0."""
        import numpy as np
        ch = as_c_history(h)
        shards = (abi.CLkShard * max(1, h.n_shards))()
        res = abi.CLkResult()
        cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32) if witness else None
        nl = abi.n_ok_lookups(h)
        lr = np.zeros(max(1, nl), np.int32) if witness else None
        rc = lib().jtb_check_lookup_witness(self._h, C.addressof(ch), max_nodes, max_rounds, max_repairs, max_lifts,
                                            flags, cr.ctypes.data if witness else None,
                                            lr.ctypes.data if witness else None, C.addressof(shards),
                                            C.addressof(res))
        if rc != 0:
            raise NativeError(f"jtb_check_lookup_witness rc={rc}: {self._err()}")
        return abi.lk_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None,
                              lr[:nl].copy() if witness else None)

    def final_configs(self, h: FlatHistory, model: CModel, shard: int = 0, cap: int = 10) -> dict:
        """knossos' :configs of an INVALID shard (`jtb_final_configs`): call directly after `check_linearizable`
        on the same history.  Returns {"total": all such configurations, "configs": the first `cap` of them}."""
        ch = as_c_history(h)
        buf = (abi.CFinalConfig * max(cap, 1))()
        total = C.c_int64(0)
        rc = lib().jtb_final_configs(self._h, C.addressof(ch), C.addressof(model), shard, C.addressof(buf), cap,
                                     C.addressof(total))
        if rc != 0:
            raise NativeError(f"jtb_final_configs rc={rc}: {self._err()}")
        return {"total": total.value, "configs": abi.final_configs_to_list(buf, min(cap, total.value))}

    def stats(self) -> dict:
        out = (C.c_ulonglong * 24)()
        lib().jtb_get_stats(C.c_void_p(self._h), out, 24)
        names = ["configs", "probes", "expansions", "ring_tail", "ring_head", "idle_polls",
                 "max_probe_len", "table_slots", "grid", "ring_entries", "attempts", "kernel_us",
                 "h2d_bytes", "d2h_bytes", "kernel_launches", "scout_steps", "scout_configs",
                 "scout_decided", "scouts", "engine_level", "beam_levels", "beam_configs", "beam_decided", "beam_attempts"]
        return {n: int(out[i]) for i, n in enumerate(names)}

    # ---- SURVEY 8(f) N2: independent/subhistory and ledger->bank on the device ------------------------------
    def partition_by_key(self, event_key) -> dict:
        """Stable partition of the events by key: {"order", "shard_off", "key_ids"} (numpy arrays)."""
        import numpy as np
        k = np.ascontiguousarray(event_key, dtype=np.int64)
        n = int(k.shape[0])
        cap = max(1, n)
        order = np.empty(n, dtype=np.int32)
        off = np.empty(cap + 1, dtype=np.int64)
        ids = np.empty(cap, dtype=np.int64)
        nk = C.c_int32(0)
        rc = lib().jtb_partition_by_key(self._h, C.c_int64(n), k.ctypes.data_as(C.c_void_p), order.ctypes.data_as(C.c_void_p),
                                        off.ctypes.data_as(C.c_void_p), ids.ctypes.data_as(C.c_void_p), C.c_int32(cap), C.byref(nk))
        if rc != 0:
            raise NativeError(f"jtb_partition_by_key rc={rc}: {self._err()}")
        return {"order": order, "shard_off": off[:nk.value + 1].copy(), "key_ids": ids[:nk.value].copy()}

    def ledger_balances(self, credits_posted, debits_posted):
        import numpy as np
        c = np.ascontiguousarray(credits_posted, dtype=np.int64)
        d = np.ascontiguousarray(debits_posted, dtype=np.int64)
        out = np.empty(c.shape[0], dtype=np.int32)
        rc = lib().jtb_ledger_balances(self._h, C.c_int64(c.shape[0]), c.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p),
                                       out.ctypes.data_as(C.c_void_p))
        if rc != 0:
            raise NativeError(f"jtb_ledger_balances rc={rc}: {self._err()}")
        return out

    # ---- K2 microbenchmark ----------------------------------------------------------------------
    def table_bench(self, n_keys: int, variant: int = 0, rounds: int = 3) -> dict:
        ins, prb, found = C.c_double(), C.c_double(), C.c_uint64()
        rc = lib().jtb_table_bench(self._h, n_keys, variant, rounds, C.addressof(ins),
                                   C.addressof(prb), C.addressof(found))
        if rc != 0:
            raise NativeError(f"jtb_table_bench rc={rc}: {self._err()}")
        return {"insert_seconds": ins.value, "probe_seconds": prb.value, "found": found.value,
                "n_keys": n_keys, "rounds": rounds, "variant": variant}


class MultiContext:
    """`jtb_multi`: the in-library multi-GPU fan-out (one process, n_gpus devices, one NCCL all-reduce(MAX) of the
    per-shard verdict vector) — what a single-process JVM host binds instead of `independent/checker`'s thread pool."""

    def __init__(self, n_gpus: int = 0, table_bytes: int = 0, max_configs: int = 0, time_budget_ms: int = 0,
                 eager_reads: bool = True, scouts: bool = True) -> None:
        L = lib()
        flags = (0 if eager_reads else abi.OPT_NO_EAGER_READS) | (0 if scouts else abi.OPT_NO_SCOUTS)
        opts = abi.COpts(0, flags, table_bytes, max_configs, time_budget_ms, 0)
        self._h = L.jtb_multi_create(C.byref(opts), n_gpus)
        if not self._h:
            raise NativeError(f"jtb_multi_create failed: {L.jtb_multi_create_error().decode()}")
        self.n_gpus = L.jtb_multi_n_gpus(self._h)

    def close(self) -> None:
        if getattr(self, "_h", None):
            lib().jtb_multi_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def check_linearizable(self, h: FlatHistory, model: CModel) -> dict:
        ch = as_c_history(h)
        shards = (abi.CLinShard * h.n_shards)()
        res = abi.CLinResult()
        dev = (C.c_int32 * max(1, h.n_shards))()
        rc = lib().jtb_multi_check_linearizable(self._h, C.addressof(ch), C.addressof(model), C.addressof(shards),
                                                C.addressof(res), C.addressof(dev))
        if rc != 0:
            raise NativeError(f"jtb_multi_check_linearizable rc={rc}: {lib().jtb_multi_last_error(self._h).decode()}")
        return {
            "valid": res.valid, "n_failures": res.n_failures, "configs": res.configs_explored, "probes": res.probes,
            "hbm_bytes_algorithmic": res.hbm_bytes_algorithmic, "key_bytes": res.key_bytes,
            "seconds_kernel": res.seconds_kernel, "seconds_total": res.seconds_total,
            "device_of_shard": [dev[s] for s in range(h.n_shards)],
            "shards": [{"valid": s.valid, "witness_index": s.witness_index, "previous_ok_index": s.previous_ok_index,
                        "cause": s.cause, "configs": s.configs_explored, "probes": s.probes} for s in shards],
        }

    def check_set_full(self, h: FlatHistory, linearizable: bool = True) -> dict:
        ch = as_c_history(h)
        shards = (abi.CSetFullShard * h.n_shards)()
        out = abi.CSetFullOut()
        out.shards = C.cast(shards, C.c_void_p)
        dev = (C.c_int32 * max(1, h.n_shards))()
        rc = lib().jtb_multi_check_set_full(self._h, C.addressof(ch), int(linearizable), C.addressof(out),
                                            C.addressof(dev))
        if rc != 0:
            raise NativeError(f"jtb_multi_check_set_full rc={rc}: {lib().jtb_multi_last_error(self._h).decode()}")
        fields = [f for f, _ in abi.CSetFullShard._fields_]
        return {"valid": out.valid, "n_failures": out.n_failures, "raia_valid": out.raia_valid,
                "n_suspect": out.n_suspect, "seconds_kernel": out.seconds_kernel, "seconds_total": out.seconds_total,
                "device_of_shard": [dev[s] for s in range(h.n_shards)],
                "shards": [{f: getattr(s, f) for f in fields} for s in shards]}


def gather_bench(ctx: "Context", table_bytes: int, in_flight: int = 4, wide: int = 1, iters: int = 64,
                 ctas_per_sm: int = 8, rounds: int = 3) -> dict:
    """Random 16 B gathers over a table of `table_bytes` (see `jtb_gather_bench`)."""
    sec, n = C.c_double(), C.c_uint64()
    rc = lib().jtb_gather_bench(ctx._h, table_bytes, in_flight, wide, iters, ctas_per_sm, rounds, C.addressof(sec),
                                C.addressof(n))
    if rc != 0:
        raise NativeError(f"jtb_gather_bench rc={rc}: {ctx._err()}")
    return {"table_bytes": table_bytes, "in_flight": in_flight, "wide": wide, "ctas_per_sm": ctas_per_sm,
            "probes": n.value, "seconds": sec.value, "Gprobes_s": n.value / sec.value / 1e9,
            "algo_GBps": 16 * wide * n.value / sec.value / 1e9}


def prepare_seconds(h: FlatHistory, model: CModel) -> float:
    """Host preparation time only (no GPU needed)."""
    ch = as_c_history(h)
    return lib().jtb_prepare_seconds(C.addressof(ch), C.addressof(model))


def prepare_info(h: FlatHistory, model: CModel) -> dict:
    """Host preparation only (no GPU needed): the layout the device search would use."""
    ch = as_c_history(h)
    info = (C.c_longlong * 4)()
    sec = lib().jtb_prepare_info(C.addressof(ch), C.addressof(model), C.addressof(info))
    return {"seconds": sec, "key_bytes": info[0], "slot_lanes": info[1], "max_classes": info[2], "ranks": info[3]}


def device_count() -> int:
    return lib().jtb_device_count()


def pinned_copy(a):
    """A copy of numpy array `a` in page-locked host memory (jtb_host_alloc): H2D copies of it run at the PCIe rate.
    The block is released when the returned array (and every view of it) is gone."""
    import weakref

    import numpy as np
    L = lib()
    L.jtb_host_alloc.restype = C.c_void_p
    L.jtb_host_alloc.argtypes = [C.c_size_t]
    L.jtb_host_free.argtypes = [C.c_void_p]
    ptr = L.jtb_host_alloc(max(a.nbytes, 16))
    if not ptr:
        raise NativeError("jtb_host_alloc failed")
    raw = (C.c_char * max(a.nbytes, 1)).from_address(ptr)
    base = np.frombuffer(raw, dtype=a.dtype, count=a.size)      # every view of the result keeps `base` alive
    weakref.finalize(base, L.jtb_host_free, C.c_void_p(ptr))
    out = base.reshape(a.shape)
    out[...] = a
    return out


def pin_history(h: FlatHistory) -> FlatHistory:
    """The history with its payload (the read id lists: the bulk of a set-full history) in page-locked memory."""
    import dataclasses
    return dataclasses.replace(h, payload=pinned_copy(h.payload))
