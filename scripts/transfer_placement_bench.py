"""Time the transfer-placement check (K12) on 10^6-op ledger-lookups histories, compare it with the TP_SEARCH CPU
oracle, and report its rounds, placed transfers and decided fraction next to the read-gap check's (K11) on the same
histories.

Workloads: the read-gap benchmark's (32 clients, tau_think 0, one quiesced final read and one quiesced final
lookup per client) at 8 and 64 accounts and p_info 0.02 and 0.  Writes one JSON document (stdout and --out) with the
card's name and power limit read in the same run, per workload K12's kernel time (CUDA events, the host's read of one
flag word per round included) and the time of the call (the library's own host clock, and the Python call around it)
of every repeat after warm-ups and their medians, the oracle's time on one CPU thread, whether the outputs are equal,
K12's rounds, placed transfers, gaps explained, unexplained, undecided, DOUBLE and LOST transfers and nodes, and K11's
gaps decided and kernel time on the device.

    python scripts/transfer_placement_bench.py --out /tmp/transfer_placement_bench.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mono_oracle  # noqa: E402
from jepsen_tigerbeetle_b200 import native, synth  # noqa: E402

FIELDS = ("valid", "n_failures", "n_reads", "n_transfers", "n_explained", "n_unexplained", "n_double", "n_lost",
          "n_undecided", "n_placed", "nodes", "rounds", "shards")


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (x.strip() for x in q.split(","))
        return {"name": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown", "power_limit": "unknown", "error": repr(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", type=int, default=1_000_000)
    ap.add_argument("--accounts", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--p-info", type=float, nargs="+", default=[0.02, 0.0])
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    doc = {"card": card(), "workloads": []}
    with native.Context(device=0) as ctx:
        for n_acct in a.accounts:
            for p_info in a.p_info:
                t0 = time.perf_counter()
                h = synth.generate_ledger_lookups(
                    synth.SynthSpec("bank", a.ops, 32, 1, p_info=p_info, tau_think_ns=0.0, n_accounts=n_acct,
                                    final_reads=True))
                gen_s = time.perf_counter() - t0
                for _ in range(a.warmup):
                    ctx.check_transfer_placement(h)
                runs, calls = [], []
                for _ in range(a.repeats):
                    t0 = time.perf_counter()
                    runs.append(ctx.check_transfer_placement(h))
                    calls.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                o = mono_oracle.check_transfer_placement(h, mono_oracle.TP_SEARCH)
                oracle_s = time.perf_counter() - t0
                k11 = ctx.check_read_gaps(h)
                g = runs[-1]
                doc["workloads"].append({
                    "ops": a.ops, "events": h.n_events, "clients": 32, "accounts": n_acct, "p_info": p_info,
                    "tau_think_ns": 0, "reads": g["n_reads"], "transfers": g["n_transfers"],
                    "explained": g["n_explained"], "unexplained": g["n_unexplained"], "double": g["n_double"],
                    "lost": g["n_lost"], "undecided": g["n_undecided"], "valid": g["valid"], "rounds": g["rounds"],
                    "placed": g["n_placed"],
                    "decided_fraction": (g["n_explained"] + g["n_unexplained"]) / max(1, g["n_reads"]),
                    "k11_decided_fraction": (k11["n_explained"] + k11["n_unexplained"]) / max(1, k11["n_reads"]),
                    "k11_undecided": k11["n_undecided"],
                    "nodes": g["nodes"], "nodes_per_gap": g["nodes"] / max(1, g["n_reads"]),
                    "seconds_kernel": [r["seconds_kernel"] for r in runs],
                    "seconds_total": [r["seconds_total"] for r in runs],
                    "seconds_call": calls,
                    "median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in runs),
                    "median_seconds_total": statistics.median(r["seconds_total"] for r in runs),
                    "median_seconds_call": statistics.median(calls),
                    "k11_seconds_kernel": k11["seconds_kernel"],
                    "oracle_tp_search_seconds": oracle_s,
                    "equal": all({k: r[k] for k in FIELDS} == {k: o[k] for k in FIELDS} for r in runs),
                    "generate_seconds": gen_s,
                })
                print(json.dumps(doc["workloads"][-1]), flush=True)
    doc["card_after"] = card()
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
