"""ctypes binding of tests/native/libjtb_hostwalk_dups.so — TEST INFRASTRUCTURE / MEASUREMENT: the level-synchronous host
walk (hostwalk.walk_bfs) with per-level statistics of how many of a level's children repeat a key generated from the
same block of W consecutive parents (what a tile filter over tiles of W parents would drop)."""
import ctypes as C
import os
import subprocess

from jepsen_tigerbeetle_b200.history import as_c_history

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SO = os.path.join(_HERE, "native", "libjtb_hostwalk_dups.so")
_SRCS = [os.path.join(_HERE, "native", "hostwalk_dups.cpp"),
         os.path.join(_ROOT, "jepsen_tigerbeetle_b200", "csrc", "jtb_prep.cpp")]
_DEPS = _SRCS + [os.path.join(_ROOT, "jepsen_tigerbeetle_b200", "csrc", f) for f in ("jtb_prep.h", "jtb_expand.h")] + \
        [os.path.join(_ROOT, "include", "jtb_check.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or any(os.path.getmtime(d) > os.path.getmtime(_SO) for d in _DEPS):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", _SO] + _SRCS)
        _lib = C.CDLL(_SO)
    return _lib


def walk_dups(h, model, windows=(32, 256, 2048), eager_reads=False, max_configs=0, level_cap=20000):
    """-> {"valid", "configs", "levels", "rows"}; rows[l] = {"parents", "children", "new", "dups": {W: count}} for the
    level expanded l-th (its parents are the configurations at depth l)."""
    ch = as_c_history(h)
    n = h.n_shards
    nw = len(windows)
    valid = (C.c_int32 * n)()
    configs, nl = C.c_ulonglong(0), C.c_int(0)
    win = (C.c_int * max(1, nw))(*windows)
    stats = (C.c_ulonglong * (level_cap * (3 + nw)))()
    rc = lib().jtb_hostwalk_dups(C.byref(ch), C.byref(model), int(eager_reads), C.c_ulonglong(max_configs), valid,
                                 C.byref(configs), win, nw, stats, level_cap, C.byref(nl))
    if rc != 0:
        raise RuntimeError(f"jtb_hostwalk_dups rc={rc}")
    rows = []
    for lv in range(min(level_cap, nl.value)):
        r = stats[lv * (3 + nw):(lv + 1) * (3 + nw)]
        rows.append({"parents": r[0], "children": r[1], "new": r[2], "dups": dict(zip(windows, r[3:]))})
    return {"valid": max(valid) if n else 0, "configs": configs.value, "levels": nl.value, "rows": rows}
