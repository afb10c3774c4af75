"""K18: the device reader of stored ledger histories against the Python path (edn.read_history + flatten_ops).

Generates 1e5- and 1e6-op ledger histories from a seed (the reference's final phase: 32 clients, one :final? read and
one :final? lookup per client returning every committed transfer), writes them as history.edn in memory, and times
`Context.read_ledger_edn` for each ledger form: the call (bytes in host memory to a FlatHistory in host memory) and
its kernels (CUDA events), each the median of 5 calls after 2 warm-ups, with the call split into the copy of the text
to the device, the kernels and the copy back.  Input GB/s is over kernel time.  The Python path is timed once: at 1e5
ops edn.read_history plus flatten_ops, at 1e6 ops flatten_ops on the generated op maps (the EDN parse there is not
run).  Outputs are compared array by array at both sizes.  Prints one JSON line per (size, form) and the card.

    python scripts/edn_read_bench.py [--sizes 100000 1000000] [--forms bank ...] [--out edn_read_bench.json]
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

from jepsen_tigerbeetle_b200 import edn, native, stored, synth  # noqa: E402
from jepsen_tigerbeetle_b200 import history as H  # noqa: E402

FORMS = ("bank", "ledger-counters", "ledger-lookups")
ARRAYS = ("type", "f", "flags", "process", "index", "time_ns", "a", "b", "c", "payload_off", "payload_len", "payload",
          "shard_off", "key_ids")


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def equal(g, p) -> bool:
    same = all(getattr(g, n).dtype == getattr(p, n).dtype and np.array_equal(getattr(g, n), getattr(p, n))
               for n in ARRAYS)
    return same and g.meta.get("multi_transfer_txns") == p.meta.get("multi_transfer_txns")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--forms", nargs="+", default=list(FORMS), choices=FORMS)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    info = card()
    print(json.dumps(info), flush=True)
    rows = []
    with native.Context(device=0) as ctx:
        for n_ops in args.sizes:
            spec = synth.SynthSpec("bank", n_ops, 32, args.seed, p_info=0.02, tau_think_ns=10e6, final_reads=True)
            t0 = time.perf_counter()
            ops = stored.generate_ledger_ops(spec, nemesis_every=1000)
            data = stored.write_edn(ops)
            gen_s = time.perf_counter() - t0
            print(json.dumps({"n_ops": n_ops, "generated_s": gen_s, "edn_bytes": len(data)}), flush=True)
            parse_s = None
            if n_ops <= 100_000:
                t0 = time.perf_counter()
                ops_read = edn.read_history(data.decode())
                parse_s = time.perf_counter() - t0
            else:
                ops_read = ops
            for form in args.forms:
                t0 = time.perf_counter()
                p = H.flatten_ops(ops_read, form)
                flat_s = time.perf_counter() - t0
                print(json.dumps({"n_ops": n_ops, "form": form, "python_flatten_s": flat_s}), flush=True)
                calls = []
                for k in range(7):
                    tm: dict = {}
                    t0 = time.perf_counter()
                    g = ctx.read_ledger_edn(data, form, timings=tm)
                    tm["call"] = time.perf_counter() - t0
                    if k >= 2:
                        calls.append(tm)
                    if k < 6:
                        del g
                med = {key: statistics.median(c[key] for c in calls)
                       for key in ("call", "seconds_h2d", "seconds_kernel", "seconds_d2h", "seconds_total")}
                row = {"n_ops": n_ops, "ops_written": len(ops), "edn_bytes": len(data), "form": form,
                       "n_events": g.n_events, "n_payload": int(g.payload.shape[0]), "equal": equal(g, p),
                       "call_s": med["call"], "h2d_s": med["seconds_h2d"], "kernel_s": med["seconds_kernel"],
                       "d2h_s": med["seconds_d2h"], "library_total_s": med["seconds_total"],
                       "input_GBps_kernel": len(data) / med["seconds_kernel"] / 1e9,
                       "python_read_history_s": parse_s if parse_s is not None else "not run",
                       "python_flatten_s": flat_s, "generate_and_write_s": gen_s, **info}
                rows.append(row)
                print(json.dumps(row), flush=True)
                del g, p
            del ops, ops_read, data
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
