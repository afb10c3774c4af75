"""K19: the host checks of a ledger compose on a stored history.edn, on the device and in Python.

Generates 1e5- and 1e6-op ledger histories from a seed as scripts/edn_read_bench.py does (32 clients, p_info 0.02, a
nemesis op every 1,000 client ops, the final phase with one :final? lookup per client returning every committed
transfer), writes them as history.edn in memory, and times:
  - `Context.ledger_edn_checks`: the call (bytes in host memory to the summary in host memory), split into the copy of
    the text to the device, the kernels (CUDA events) and the copy back, each the median of 5 calls after 2 warm-ups;
  - `ledger_checker(linear=False).check` end to end on a `StoredLedgerHistory` (once; it reads the "bank" form and the
    summary on the device);
  - at 1e5 ops only, the Python path: edn.read_history plus the four checkers (unexpected-ops, lookup-transfers,
    final-reads, stats), once.
At 1e5 ops the four checkers' results on the StoredLedgerHistory must equal the Python path's, op maps included.  At
1e6 ops (the EDN parse would take about 10 minutes) the verdicts, counts and the ordinals of the flagged ops are
compared with the four checkers run on the generated op maps, without reading the flagged ops' bytes.  Prints the card
and one JSON line per size.

    python scripts/edn_checks_bench.py [--sizes 100000 1000000] [--out edn_checks_bench.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from jepsen_tigerbeetle_b200 import checker as CK  # noqa: E402
from jepsen_tigerbeetle_b200 import edn, native, stored, synth  # noqa: E402

CHECKERS = {"unexpected-ops": CK.UnexpectedOps(), "lookup-transfers": CK.LookupAllInvokedTransfers(),
            "final-reads": CK.FinalReads(), "stats": CK.Stats()}


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return {"gpu": name, "power_limit": power}


def ordinals(ops) -> dict:
    """op -> its ordinal, for the op maps the checkers return"""
    return {id(op): k for k, op in enumerate(ops)}


def shape(r: dict, where) -> dict:
    """A checker's result with every op replaced by its ordinal (`where` maps an op to it) and sets by their size."""
    out = {}
    for k, v in r.items():
        if k in ("open-ops",):
            out[k] = [[ms, where(op)] for ms, op in v]
        elif k in ("fail-ops", "suspect-final-lookups"):
            out[k] = [where(op) for op in v]
        elif k.startswith("unequal-"):
            out[k] = len(v)
        else:
            out[k] = v
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--seed", type=int, default=1)
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
            calls = []
            for k in range(7):
                t0 = time.perf_counter()
                s = ctx.ledger_edn_checks(data)
                t = time.perf_counter() - t0
                assert s["refused"] is None, s["refused"]
                if k >= 2:
                    calls.append(dict(s, call=t))
            med = {key: statistics.median(c[key] for c in calls)
                   for key in ("call", "seconds_h2d", "seconds_kernel", "seconds_d2h", "seconds_total")}

            h = CK.StoredLedgerHistory(data, ctx=ctx)
            t0 = time.perf_counter()
            composed = CK.ledger_checker(ctx=ctx, linear=False).check({}, h)
            compose_s = time.perf_counter() - t0
            device = {name: c.check({}, h) for name, c in CHECKERS.items()}
            python_s = parse_s = None
            if n_ops <= 100_000:
                t0 = time.perf_counter()
                ops_read = edn.read_history(data.decode())
                parse_s = time.perf_counter() - t0
                t0 = time.perf_counter()
                python = {name: c.check({}, ops_read) for name, c in CHECKERS.items()}
                python_s = time.perf_counter() - t0
                equal = device == python
            else:   # the checkers on the generated op maps; the device's ops by the ordinal of their bytes
                python = {name: c.check({}, ops) for name, c in CHECKERS.items()}
                begin = {int(r["begin"]): int(r["op"]) for kind in ("open", "fails", "final_lookups")
                         for r in s[kind]}
                pos = ordinals(ops)
                equal = all(shape(device[n], lambda op: begin[op._begin]) == shape(python[n], lambda op: pos[id(op)])
                            for n in CHECKERS)
            row = {"n_ops": n_ops, "ops_written": len(ops), "edn_bytes": len(data), "equal": equal,
                   "verdicts": {n: r["valid?"] for n, r in device.items()}, "compose_valid": composed["valid?"],
                   **{k: s[k] for k in ("n_client", "n_open", "n_fail", "n_final_reads", "n_final_lookups",
                                        "n_read_classes", "n_lookup_classes", "n_invoked", "n_suspect")},
                   "call_s": med["call"], "h2d_s": med["seconds_h2d"], "kernel_s": med["seconds_kernel"],
                   "d2h_s": med["seconds_d2h"], "library_total_s": med["seconds_total"],
                   "input_GBps_kernel": len(data) / med["seconds_kernel"] / 1e9, "compose_s": compose_s,
                   "python_read_history_s": parse_s if parse_s is not None else "not run",
                   "python_checkers_s": python_s if python_s is not None else "not run",
                   "generate_and_write_s": gen_s, **info}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del ops, data, h, s, calls, device, python, composed
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
