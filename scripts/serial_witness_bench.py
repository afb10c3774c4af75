"""Time the serial-witness check (K13) on the transfer-placement benchmark's 10^6-op ledger-lookups histories and on
the C3 instance, next to the transfer-placement check (K12) in the same run, and compare it with the SW_SEARCH CPU
oracle.

Workloads: K12's four (32 clients, tau_think 0, one quiesced final read and one quiesced final lookup per client; 8 and
64 accounts x p_info 0 and 0.02) and C3 (10,000 ops, 32 clients, seed 1, p_info 0.02).  Writes one JSON document
(stdout and --out) with the card's name and power limit read in the same run and, per workload, K13's and K12's
kernel time (CUDA events; K13's includes K12's stage) and the time of the Python call around them, every repeat after
the warm-ups and their medians, K13's witness rounds, verdict and causes, committed crashed transfers, the oracle's
time on one CPU thread, and whether the device equals the oracle (commit_read included).

    python scripts/serial_witness_bench.py --out /tmp/serial_witness_bench.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mono_oracle  # noqa: E402
from jepsen_tigerbeetle_b200 import abi, native, synth  # noqa: E402

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_committed", "n_committed_crashed", "n_after", "nodes",
          "rounds", "shards")


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in q.split(","))
        return {"name": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown", "power_limit": "unknown", "error": repr(e)}


def timed(fn, warmup: int, repeats: int):
    for _ in range(warmup):
        fn()
    runs, calls = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        runs.append(fn())
        calls.append(time.perf_counter() - t0)
    return runs, calls


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true", help="skip SW_SEARCH (minutes per 10^6-op history)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    loads = [(a.ops, n, p, 0.0) for n in (8, 64) for p in (0.0, 0.02)] + [(10_000, 8, 0.02, None)]
    doc = {"card": card(), "workloads": []}
    with native.Context(device=0) as ctx:
        for ops, n_acct, p_info, tau in loads:
            kw = {} if tau is None else {"tau_think_ns": tau}
            h = synth.generate_ledger_lookups(synth.SynthSpec("bank", ops, 32, 1, p_info=p_info, n_accounts=n_acct,
                                                              final_reads=True, **kw))
            sw, sw_calls = timed(lambda: ctx.check_serial_witness(h, witness=True), a.warmup, a.repeats)
            tp, tp_calls = timed(lambda: ctx.check_transfer_placement(h), a.warmup, a.repeats)
            g = sw[-1]
            w = {"workload": "C3" if tau is None else "K12", "ops": ops, "accounts": n_acct, "p_info": p_info,
                 "reads": g["n_reads"], "transfers": g["n_transfers"], "valid": g["valid"],
                 "causes": sorted({abi.CAUSE_NAME[s["cause"]] or "none" for s in g["shards"]}),
                 "witness_rounds": g["rounds"], "witness_nodes": g["nodes"], "committed": g["n_committed"],
                 "committed_crashed": g["n_committed_crashed"], "after": g["n_after"],
                 "k12_valid": tp[-1]["valid"], "k12_undecided": tp[-1]["n_undecided"],
                 "median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in sw),
                 "median_seconds_call": statistics.median(sw_calls),
                 "k12_median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in tp),
                 "k12_median_seconds_call": statistics.median(tp_calls),
                 "seconds_kernel": [r["seconds_kernel"] for r in sw], "seconds_call": sw_calls,
                 "k12_seconds_kernel": [r["seconds_kernel"] for r in tp], "k12_seconds_call": tp_calls,
                 "repeats_equal": all({k: r[k] for k in FIELDS} == {k: g[k] for k in FIELDS} and
                                      np.array_equal(r["commit_read"], g["commit_read"]) for r in sw)}
            if not a.no_oracle:
                t0 = time.perf_counter()
                o = mono_oracle.check_serial_witness(h)
                w["oracle_sw_search_seconds"] = time.perf_counter() - t0
                w["equal"] = ({k: g[k] for k in FIELDS} == {k: o[k] for k in FIELDS} and
                              bool(np.array_equal(g["commit_read"], o["commit_read"])))
            doc["workloads"].append(w)
            print(json.dumps(w), flush=True)
    doc["card_after"] = card()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
