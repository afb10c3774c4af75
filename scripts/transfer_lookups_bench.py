"""Time the transfer-lookup check (K9) on 10^6-op ledger histories and compare it with the TL_SWEEP CPU oracle.

Workloads: 32 clients, tau_think 0, p_info 0.02, one quiesced final read and one quiesced final lookup per client, at 8
and 64 accounts (with --lost also the same histories with one lost :ok transfer).  Writes one JSON document (stdout and
--out) with the card's name and power limit read in the same run, per workload the kernel time (CUDA events) and the
time of the call (the library's own host clock, and the Python call around it) of every repeat after warm-ups and their
medians, the oracle's times on the same arrays (same warm-ups and repeats) and whether the outputs are equal.

    python scripts/transfer_lookups_bench.py --out /tmp/transfer_lookups_bench.json
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

FIELDS = ("valid", "n_failures", "n_lookups", "n_records", "n_transfers", "n_reads", "n_violations", "shards")


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
    ap.add_argument("--lost", action="store_true", help="also time the lost-transfer variant of every workload")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    doc = {"card": card(), "workloads": []}
    with native.Context(device=0) as ctx:
        for n_acct in a.accounts:
            for lost in ((False, True) if a.lost else (False,)):
                t0 = time.perf_counter()
                h = synth.generate_ledger_lookups(
                    synth.SynthSpec("bank", a.ops, 32, 1, p_info=0.02, tau_think_ns=0.0, n_accounts=n_acct,
                                    final_reads=True), lost_transfer=lost)
                gen_s = time.perf_counter() - t0
                for _ in range(a.warmup):
                    ctx.check_transfer_lookups(h)
                runs, calls = [], []
                for _ in range(a.repeats):
                    t0 = time.perf_counter()
                    runs.append(ctx.check_transfer_lookups(h))
                    calls.append(time.perf_counter() - t0)
                for _ in range(a.warmup):
                    mono_oracle.check_transfer_lookups(h, mono_oracle.TL_SWEEP)
                oracle_s = []
                for _ in range(a.repeats):
                    t0 = time.perf_counter()
                    o = mono_oracle.check_transfer_lookups(h, mono_oracle.TL_SWEEP)
                    oracle_s.append(time.perf_counter() - t0)
                g = runs[-1]
                doc["workloads"].append({
                    "ops": a.ops, "events": h.n_events, "clients": 32, "accounts": n_acct, "lost_transfer": lost,
                    "p_info": 0.02, "tau_think_ns": 0, "reads": g["n_reads"], "transfers": g["n_transfers"],
                    "lookups": g["n_lookups"], "records": g["n_records"], "payload_bytes": int(h.payload.nbytes),
                    "violations": g["n_violations"], "valid": g["valid"], "kind": g["shards"][0]["kind"],
                    "seconds_kernel": [r["seconds_kernel"] for r in runs],
                    "seconds_total": [r["seconds_total"] for r in runs],
                    "seconds_call": calls,
                    "median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in runs),
                    "median_seconds_total": statistics.median(r["seconds_total"] for r in runs),
                    "median_seconds_call": statistics.median(calls),
                    "oracle_tl_sweep_seconds": oracle_s, "median_oracle_tl_sweep_seconds": statistics.median(oracle_s),
                    "oracle_valid": o["valid"],
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
