"""ctypes binding of the monotonic-key and counter-bounds CPU oracles (libjtb_mono_oracle.so).  TEST INFRASTRUCTURE
ONLY.

MONO_GRAPH builds Elle's monotonic-key graph literally (plus real-time edges) and runs Tarjan; MONO_PAIRS searches
for 2-cycles by brute force.  See mono_oracle.cpp.  CB_LITERAL sums every transfer for every (read, key); CB_SWEEP
keeps running sums over one walk of the events.  See counter_bounds.cpp.  TL_LITERAL checks every (lookup, transfer)
pair and every (read, key, lookup) triple; TL_SWEEP walks with hash maps, sorted M lists, prefix maxima and suffix
minima.  See transfer_lookups.cpp.  RX_BRUTE enumerates every subset of a read's "may" transfers; RX_SEARCH is the
library's budgeted pruning and depth-first search over a sweep.  See read_explanations.cpp.  RG_BRUTE enumerates every
subset of a gap's eligible transfers; RG_SEARCH is the library's amount filter, caps and search per gap.  See
read_gaps.cpp.  TP_BRUTE enumerates every placement of each transfer in a gap of its window; TP_SEARCH is the
library's rounds of per-gap searches with owned transfers carried between gaps.  See transfer_placement.cpp.
SW_SEARCH is TP_SEARCH followed by the library's witness rounds, real-time pass and commit_read.  See
serial_witness.cpp.  RW_SEARCH is SW_SEARCH followed by the library's repair rounds.  See repaired_witness.cpp.
LW_SEARCH is RW_SEARCH with lift steps where its repairs would stop.  See lifted_witness.cpp and repair_common.h.
CW_SEARCH is LW_SEARCH followed by the library's class pass on the shards it leaves unproved.  See class_witness.cpp.
LK_SEARCH is CW_SEARCH followed by the library's placement of the lookups; LK_BRUTE is its definition on tiny
histories.  See lookup_witness.cpp."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

from jepsen_tigerbeetle_b200 import abi
from jepsen_tigerbeetle_b200.history import FlatHistory, as_c_history

MONO_GRAPH, MONO_PAIRS = 0, 1
CB_LITERAL, CB_SWEEP = 0, 1
TL_LITERAL, TL_SWEEP = 0, 1
RX_BRUTE, RX_SEARCH = 0, 1
RG_BRUTE, RG_SEARCH = 0, 1
TP_BRUTE, TP_SEARCH = 0, 1
SW_SEARCH = 1
RW_SEARCH = 1
LW_SEARCH = 1
CW_SEARCH = 1
LK_BRUTE, LK_SEARCH = 0, 1
DECIDE_PARTIAL = 1 << 16   # decide shards with partial reads instead of reporting them UNKNOWN
_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
    """The library in mono_oracle/, rebuilt when stale; when the directory is read-only a rebuild goes to a fresh
    temporary directory instead."""
    so = os.path.join(_HERE, "libjtb_mono_oracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("mono_oracle.cpp", "counter_bounds.cpp", "transfer_lookups.cpp",
                                                "read_explanations.cpp", "read_gaps.cpp", "transfer_placement.cpp",
                                                "serial_witness.cpp", "repaired_witness.cpp", "lifted_witness.cpp",
                                                "class_witness.cpp", "lookup_witness.cpp", "gaps_common.h", "witness_common.h",
                                                "repair_common.h", "Makefile")]
    srcs.append(os.path.join(_HERE, "..", "include", "jtb_check.h"))
    stale = not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        if not os.access(_HERE, os.W_OK):
            so = os.path.join(tempfile.mkdtemp(prefix="jtb_mono_oracle_"), "libjtb_mono_oracle.so")
            subprocess.check_call(["make", "-C", _HERE, "-B", "-s", f"LIB={so}"], stdout=subprocess.DEVNULL)
            return so
        subprocess.check_call(["make", "-C", _HERE, "-B", "-s"], stdout=subprocess.DEVNULL)
    return so


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.jtbm_last_error.restype = C.c_char_p
        _LIB.jtbm_check_monotonic_keys.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        _LIB.jtbm_cb_last_error.restype = C.c_char_p
        _LIB.jtbm_check_counter_bounds.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        _LIB.jtbm_tl_last_error.restype = C.c_char_p
        _LIB.jtbm_check_transfer_lookups.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        _LIB.jtbm_rx_last_error.restype = C.c_char_p
        _LIB.jtbm_check_read_explanations.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p,
                                                      C.c_void_p, C.c_void_p]
        _LIB.jtbm_rg_last_error.restype = C.c_char_p
        _LIB.jtbm_check_read_gaps.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                              C.c_void_p]
        _LIB.jtbm_tp_last_error.restype = C.c_char_p
        _LIB.jtbm_check_transfer_placement.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                                       C.c_void_p, C.c_void_p]
        _LIB.jtbm_sw_last_error.restype = C.c_char_p
        _LIB.jtbm_check_serial_witness.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.jtbm_rw_last_error.restype = C.c_char_p
        _LIB.jtbm_check_repaired_witness.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                                     C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.jtbm_lw_last_error.restype = C.c_char_p
        _LIB.jtbm_check_lifted_witness.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                                   C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.jtbm_cw_last_error.restype = C.c_char_p
        _LIB.jtbm_check_class_witness.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                                  C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB.jtbm_lk_last_error.restype = C.c_char_p
        _LIB.jtbm_check_lookup_witness.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                                   C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]
    return _LIB


def check_monotonic_keys(h: FlatHistory, algo: int = MONO_GRAPH, realtime: bool = True,
                         decide_partial: bool = False) -> dict:
    """Twin of `jtb_check_monotonic_keys` (same result dict as `native.Context.check_monotonic_keys`)."""
    ch = as_c_history(h)
    shards = (abi.CMonoShard * max(1, h.n_shards))()
    res = abi.CMonoResult()
    flags = (0 if realtime else abi.MONO_NO_REALTIME) | (DECIDE_PARTIAL if decide_partial else 0)
    rc = lib().jtbm_check_monotonic_keys(C.addressof(ch), flags, algo, C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_last_error().decode())
    return abi.mono_to_dict(res, shards[:h.n_shards])


def check_counter_bounds(h: FlatHistory, algo: int = CB_SWEEP, flags: int = 0) -> dict:
    """Twin of `jtb_check_counter_bounds` (same result dict as `native.Context.check_counter_bounds`)."""
    ch = as_c_history(h)
    shards = (abi.CCbShard * max(1, h.n_shards))()
    res = abi.CCbResult()
    rc = lib().jtbm_check_counter_bounds(C.addressof(ch), flags, algo, C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_cb_last_error().decode())
    return abi.cb_to_dict(res, shards[:h.n_shards])


def check_transfer_lookups(h: FlatHistory, algo: int = TL_SWEEP, flags: int = 0) -> dict:
    """Twin of `jtb_check_transfer_lookups` (same result dict as `native.Context.check_transfer_lookups`)."""
    ch = as_c_history(h)
    shards = (abi.CTlShard * max(1, h.n_shards))()
    res = abi.CTlResult()
    rc = lib().jtbm_check_transfer_lookups(C.addressof(ch), flags, algo, C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_tl_last_error().decode())
    return abi.tl_to_dict(res, shards[:h.n_shards])


def check_read_explanations(h: FlatHistory, algo: int = RX_SEARCH, max_nodes: int = 0, flags: int = 0,
                            per_read: bool = False) -> dict:
    """Twin of `jtb_check_read_explanations` (same result dict as `native.Context.check_read_explanations`).
    per_read=True adds "per_read": one code per :ok read in shard-major completion order (0 explained, 1 KEY, 2 JOINT,
    3 undecided)."""
    import numpy as np
    ch = as_c_history(h)
    shards = (abi.CRxShard * max(1, h.n_shards))()
    res = abi.CRxResult()
    codes = np.zeros(max(1, int(np.count_nonzero(h.f == 0))), np.int8)
    rc = lib().jtbm_check_read_explanations(C.addressof(ch), max_nodes, flags, algo, C.addressof(shards),
                                            C.addressof(res), codes.ctypes.data if per_read else None)
    if rc != 0:
        raise RuntimeError(lib().jtbm_rx_last_error().decode())
    out = abi.rx_to_dict(res, shards[:h.n_shards])
    if per_read:
        out["per_read"] = codes[:res.n_reads].tolist()
    return out


def check_read_gaps(h: FlatHistory, algo: int = RG_SEARCH, max_nodes: int = 0, flags: int = 0,
                    per_gap: bool = False) -> dict:
    """Twin of `jtb_check_read_gaps` (same result dict as `native.Context.check_read_gaps`).  per_gap=True adds
    "per_gap": one code per :ok read in shard-major order, a full-key shard's gaps in gap order (0 explained, 1 KEY,
    2 JOINT, 3 undecided; 3 for every read of a partial-read shard)."""
    import numpy as np
    ch = as_c_history(h)
    shards = (abi.CRgShard * max(1, h.n_shards))()
    res = abi.CRgResult()
    codes = np.zeros(max(1, int(np.count_nonzero(h.f == 0))), np.int8)
    rc = lib().jtbm_check_read_gaps(C.addressof(ch), max_nodes, flags, algo, C.addressof(shards), C.addressof(res),
                                    codes.ctypes.data if per_gap else None)
    if rc != 0:
        raise RuntimeError(lib().jtbm_rg_last_error().decode())
    out = abi.rg_to_dict(res, shards[:h.n_shards])
    if per_gap:
        out["per_gap"] = codes[:res.n_reads].tolist()
    return out


def check_transfer_placement(h: FlatHistory, algo: int = TP_SEARCH, max_nodes: int = 0, max_rounds: int = 0,
                             flags: int = 0) -> dict:
    """Twin of `jtb_check_transfer_placement` (same result dict as `native.Context.check_transfer_placement`).
    TP_BRUTE fills only the verdict, the cause and the read and transfer counts."""
    ch = as_c_history(h)
    shards = (abi.CTpShard * max(1, h.n_shards))()
    res = abi.CTpResult()
    rc = lib().jtbm_check_transfer_placement(C.addressof(ch), max_nodes, max_rounds, flags, algo,
                                             C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_tp_last_error().decode())
    return abi.tp_to_dict(res, shards[:h.n_shards])


def check_serial_witness(h: FlatHistory, algo: int = SW_SEARCH, max_nodes: int = 0, max_rounds: int = 0,
                         flags: int = 0, witness: bool = True) -> dict:
    """Twin of `jtb_check_serial_witness` (same result dict as `native.Context.check_serial_witness`)."""
    import numpy as np
    ch = as_c_history(h)
    shards = (abi.CSwShard * max(1, h.n_shards))()
    res = abi.CSwResult()
    cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32)
    rc = lib().jtbm_check_serial_witness(C.addressof(ch), max_nodes, max_rounds, flags, algo,
                                         cr.ctypes.data if witness else None, C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_sw_last_error().decode())
    return abi.witness_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)


def check_repaired_witness(h: FlatHistory, algo: int = RW_SEARCH, max_nodes: int = 0, max_rounds: int = 0,
                           max_repairs: int = 0, flags: int = 0, witness: bool = True) -> dict:
    """Twin of `jtb_check_repaired_witness` (same result dict as `native.Context.check_repaired_witness`)."""
    import numpy as np
    ch = as_c_history(h)
    shards = (abi.CRwShard * max(1, h.n_shards))()
    res = abi.CRwResult()
    cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32)
    rc = lib().jtbm_check_repaired_witness(C.addressof(ch), max_nodes, max_rounds, max_repairs, flags, algo,
                                           cr.ctypes.data if witness else None, C.addressof(shards),
                                           C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_rw_last_error().decode())
    return abi.witness_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)


def check_lifted_witness(h: FlatHistory, algo: int = LW_SEARCH, max_nodes: int = 0, max_rounds: int = 0,
                         max_repairs: int = 0, max_lifts: int = 0, flags: int = 0, witness: bool = True) -> dict:
    """Twin of `jtb_check_lifted_witness` (same result dict as `native.Context.check_lifted_witness`)."""
    import numpy as np
    ch = as_c_history(h)
    shards = (abi.CLwShard * max(1, h.n_shards))()
    res = abi.CLwResult()
    cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32)
    rc = lib().jtbm_check_lifted_witness(C.addressof(ch), max_nodes, max_rounds, max_repairs, max_lifts, flags, algo,
                                         cr.ctypes.data if witness else None, C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_lw_last_error().decode())
    return abi.witness_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)


def check_class_witness(h: FlatHistory, algo: int = CW_SEARCH, max_nodes: int = 0, max_rounds: int = 0,
                        max_repairs: int = 0, max_lifts: int = 0, flags: int = 0, witness: bool = True) -> dict:
    """Twin of `jtb_check_class_witness` (same result dict as `native.Context.check_class_witness`)."""
    import numpy as np
    ch = as_c_history(h)
    shards = (abi.CCwShard * max(1, h.n_shards))()
    res = abi.CCwResult()
    cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32)
    rc = lib().jtbm_check_class_witness(C.addressof(ch), max_nodes, max_rounds, max_repairs, max_lifts, flags, algo,
                                        cr.ctypes.data if witness else None, C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_cw_last_error().decode())
    return abi.witness_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None)


def check_lookup_witness(h: FlatHistory, algo: int = LK_SEARCH, max_nodes: int = 0, max_rounds: int = 0,
                         max_repairs: int = 0, max_lifts: int = 0, flags: int = 0, witness: bool = True) -> dict:
    """Twin of `jtb_check_lookup_witness` (same result dict as `native.Context.check_lookup_witness`).  LK_BRUTE fills
    only each shard's valid (JTB_VALID when a serial order exists, else JTB_INVALID), n_reads and n_transfers."""
    import numpy as np
    ch = as_c_history(h)
    shards = (abi.CLkShard * max(1, h.n_shards))()
    res = abi.CLkResult()
    cr = np.zeros(max(1, abi.n_transfer_records(h)), np.int32)
    nl = abi.n_ok_lookups(h)
    lr = np.zeros(max(1, nl), np.int32)
    rc = lib().jtbm_check_lookup_witness(C.addressof(ch), max_nodes, max_rounds, max_repairs, max_lifts, flags, algo,
                                         cr.ctypes.data if witness else None, lr.ctypes.data if witness else None,
                                         C.addressof(shards), C.addressof(res))
    if rc != 0:
        raise RuntimeError(lib().jtbm_lk_last_error().decode())
    return abi.witness_to_dict(res, shards[:h.n_shards], cr[:res.n_transfers].copy() if witness else None,
                               lr[:nl].copy() if witness else None)
