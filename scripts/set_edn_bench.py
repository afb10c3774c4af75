"""K20: the device reader of stored set-full histories against the Python path (edn.read_history(independent=True) +
flatten_ops(..., "set")), and the set-full workload checker on a StoredSetHistory.

Generates BASELINE's C4 shape (`synth.config_c4`: 1e5 ops, 64 clients) at K = 64 and K = 8 keys and writes it as
history.edn in memory, in the store's format: one `#jepsen.history.Op{...}` per line, `[k id]` adds, `[k nil]` read
invokes and `[k #{...}]` :ok reads whose members are shuffled, as a Clojure hash set prints them.  (The file is written
from the flat arrays, not through `stored.set_ops` + `write_edn`, which would hold the 10^8 ids of K = 8 as Python
frozensets; at K = 64 the Python path below checks that the two agree.)  Then it times `Context.read_set_edn`: the
call (bytes in host memory to a FlatHistory in host memory), the copy of the text to the device, the kernels (CUDA
events) and the copy back, each the median of 5 calls after 2 warm-ups; input GB/s is over kernel time.  It also times
one `set_full_workload_checker().check` on a fresh `StoredSetHistory` (the device read plus the two check_set_full
calls the compose makes, one for set-full and one for read-all-invoked-adds) and one check_set_full call alone, which
is what the second call costs.  The Python path (read_history + flatten_ops) runs once where --python-keys includes
K; elsewhere the arrays are compared with the generator's, spelled as flatten_ops spells them (the CPU tests check that
the two agree).  Prints the card, then one JSON line per K.

    python scripts/set_edn_bench.py [--keys 64 8] [--python-keys 64] [--out set_edn_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from jepsen_tigerbeetle_b200 import checker as CK  # noqa: E402
from jepsen_tigerbeetle_b200 import edn, native, synth  # noqa: E402
from jepsen_tigerbeetle_b200 import history as H  # noqa: E402

ARRAYS = ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_off", "payload_len", "payload",
          "shard_off", "key_ids")
TYPE_NAME = {H.T_INVOKE: "invoke", H.T_OK: "ok", H.T_FAIL: "fail", H.T_INFO: "info"}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def write_set_edn(h: H.FlatHistory, seed: int) -> bytes:
    """history.edn of a keyed set history, in history order, with each :ok read's members shuffled"""
    rng = np.random.default_rng(seed)
    key = np.repeat(h.key_ids, np.diff(h.shard_off))
    lines = []
    for e in np.argsort(h.index, kind="stable"):
        t, k = int(h.type[e]), int(key[e])
        if h.f[e] == H.F_ADD:
            f, v = "add", str(int(h.a[e]))
        else:
            f, v = "read", "nil"
            if t == H.T_OK:
                pl = h.payload[h.payload_off[e]:h.payload_off[e] + h.payload_len[e]]
                v = "#{" + " ".join(map(str, rng.permutation(pl).tolist())) + "}"
        extra = (", :error :timeout" if t == H.T_INFO else "") + (", :final? true" if h.flags[e] & H.FLAG_FINAL else "")
        lines.append(f"#jepsen.history.Op{{:index {int(h.index[e])}, :time {int(h.time_ns[e])}, :type :{TYPE_NAME[t]}, "
                     f":process {int(h.process[e])}, :f :{f}, :value [{k} {v}]{extra}}}")
    return ("\n".join(lines) + "\n").encode()


def expected(h: H.FlatHistory) -> H.FlatHistory:
    """h as flatten_ops spells it: the payload packed, adds without a payload (-1) and reads with a = 0"""
    r = h.select_shards(range(h.n_shards))
    add = r.f == H.F_ADD
    r.payload_len = np.where(add, -1, r.payload_len).astype(np.int32)
    r.a = np.where(add, r.a, 0).astype(np.int32)
    return r


def equal(g, p) -> bool:
    return all(getattr(g, n).dtype == getattr(p, n).dtype and np.array_equal(getattr(g, n), getattr(p, n))
               for n in ARRAYS)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, nargs="+", default=[64, 8])
    ap.add_argument("--python-keys", type=int, nargs="*", default=[64])
    ap.add_argument("--n-ops", type=int, default=100_000)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    with native.Context(device=0) as ctx:
        for n_keys in args.keys:
            t0 = time.perf_counter()
            h = synth.config_c4(seed=args.seed, n_keys=n_keys, n_ops=args.n_ops)
            data = write_set_edn(h, args.seed)
            gen_s = time.perf_counter() - t0
            print(json.dumps({"n_keys": n_keys, "generated_s": gen_s, "edn_bytes": len(data)}), flush=True)
            calls = []
            for k in range(7):
                tm: dict = {}
                t0 = time.perf_counter()
                g = ctx.read_set_edn(data, timings=tm)
                tm["call"] = time.perf_counter() - t0
                if k >= 2:
                    calls.append(tm)
                if k < 6:
                    del g
            med = {key: statistics.median(c[key] for c in calls)
                   for key in ("call", "seconds_h2d", "seconds_kernel", "seconds_d2h", "seconds_total")}
            checker = CK.set_full_workload_checker(ctx=ctx)
            checker.check({}, g)   # warm-up of the checks
            t0 = time.perf_counter()
            r = checker.check({}, CK.StoredSetHistory(data, ctx=ctx))
            checker_s = time.perf_counter() - t0
            one = []
            for _ in range(3):
                t0 = time.perf_counter()
                ctx.check_set_full(g, True)
                one.append(time.perf_counter() - t0)
            row = {"n_ops": args.n_ops, "n_keys": n_keys, "edn_bytes": len(data), "n_events": g.n_events,
                   "n_payload": int(g.payload.shape[0]), "call_s": med["call"], "h2d_s": med["seconds_h2d"],
                   "kernel_s": med["seconds_kernel"], "d2h_s": med["seconds_d2h"],
                   "library_total_s": med["seconds_total"], "input_GBps_kernel": len(data) / med["seconds_kernel"] / 1e9,
                   "workload_checker_s": checker_s, "workload_valid": r["valid?"],
                   "one_check_set_full_s": statistics.median(one), "generate_and_write_s": gen_s}
            if n_keys in args.python_keys:
                t0 = time.perf_counter()
                ops = edn.read_history(data.decode(), independent=True)
                row["python_read_history_s"] = time.perf_counter() - t0
                t0 = time.perf_counter()
                p = H.flatten_ops(ops, "set")
                row["python_flatten_s"] = time.perf_counter() - t0
                row["equal_python_path"] = equal(g, p)
                del ops, p
            else:
                row["python_read_history_s"] = row["python_flatten_s"] = "not run"
            row["equal_generator"] = equal(g, expected(h))
            row.update(info)
            rows.append(row)
            print(json.dumps(row), flush=True)
            del g, h, data
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
