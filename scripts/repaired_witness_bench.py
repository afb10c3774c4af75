"""Time the repaired serial witness (K14) next to the serial-witness check (K13) on K13's benchmark workloads, and
compare it with the RW_SEARCH CPU oracle.

Workloads: the four 10^6-op ledger-lookups histories (32 clients, tau_think 0, seed 1, one quiesced final read and
lookup per client; 8 and 64 accounts x p_info 0 and 0.02) and C3 (10,000 ops, 32 clients, seed 1, p_info 0.02).
Writes one JSON document (stdout and --out) with the card's name and power limit read in the same run, before and
after, and per workload: K14's verdict, causes, repair rounds, bans and witness rounds, K13's verdict and causes, both
checks' kernel time (CUDA events) and call time (every repeat after the warm-ups, and the medians), the oracle's time
on one CPU thread, and whether the device equals the oracle (commit_read included).

    python scripts/repaired_witness_bench.py --out /tmp/repaired_witness_bench.json
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import mono_oracle  # noqa: E402
from jepsen_tigerbeetle_b200 import abi, native, synth  # noqa: E402
from serial_witness_bench import card, timed  # noqa: E402

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes",
          "rounds", "repairs", "n_bans", "shards")


def causes(r) -> list:
    return sorted({abi.CAUSE_NAME[s["cause"]] or "none" for s in r["shards"]})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true", help="skip RW_SEARCH (minutes per 10^6-op history)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    loads = [(a.ops, n, p, 0.0) for n in (8, 64) for p in (0.0, 0.02)] + [(10_000, 8, 0.02, None)]
    doc = {"card": card(), "workloads": []}
    with native.Context(device=0) as ctx:
        for ops, n_acct, p_info, tau in loads:
            kw = {} if tau is None else {"tau_think_ns": tau}
            h = synth.generate_ledger_lookups(synth.SynthSpec("bank", ops, 32, 1, p_info=p_info, n_accounts=n_acct,
                                                              final_reads=True, **kw))
            rw, rw_calls = timed(lambda: ctx.check_repaired_witness(h, witness=True), a.warmup, a.repeats)
            sw, sw_calls = timed(lambda: ctx.check_serial_witness(h, witness=True), a.warmup, a.repeats)
            g, k = rw[-1], sw[-1]
            w = {"workload": "C3" if tau is None else "10^6", "ops": ops, "accounts": n_acct, "p_info": p_info,
                 "reads": g["n_reads"], "valid": g["valid"], "causes": causes(g), "repairs": g["repairs"],
                 "bans": g["n_bans"], "witness_rounds": g["rounds"], "nodes": g["nodes"],
                 "committed_crashed": g["n_committed_crashed"], "k13_valid": k["valid"], "k13_causes": causes(k),
                 "median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in rw),
                 "median_seconds_call": statistics.median(rw_calls),
                 "k13_median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in sw),
                 "k13_median_seconds_call": statistics.median(sw_calls),
                 "seconds_kernel": [r["seconds_kernel"] for r in rw], "seconds_call": rw_calls,
                 "k13_seconds_kernel": [r["seconds_kernel"] for r in sw], "k13_seconds_call": sw_calls,
                 "repeats_equal": all({f: r[f] for f in FIELDS} == {f: g[f] for f in FIELDS} and
                                      np.array_equal(r["commit_read"], g["commit_read"]) for r in rw)}
            if not a.no_oracle:
                t0 = time.perf_counter()
                o = mono_oracle.check_repaired_witness(h)
                w["oracle_rw_search_seconds"] = time.perf_counter() - t0
                w["equal"] = ({f: g[f] for f in FIELDS} == {f: o[f] for f in FIELDS} and
                              bool(np.array_equal(g["commit_read"], o["commit_read"])))
            doc["workloads"].append(w)
            print(json.dumps({x: y for x, y in w.items() if not isinstance(y, list) or x.endswith("causes")}),
                  flush=True)
    doc["card_after"] = card()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
