"""Time the lifted serial witness (K15) next to the repaired serial witness (K14), and compare it with the LW_SEARCH
CPU oracle.

Workloads: K14's five (the four 10^6-op ledger-lookups histories, 32 clients, tau_think 0, seed 1, one quiesced final
read and lookup per client, 8 and 64 accounts x p_info 0 and 0.02; and C3, 10,000 ops, 32 clients, seed 1, p_info
0.02) and the eight 10^5-op panel histories (8 and 64 accounts, p_info 0 and 0.02, seeds 1 and 2, tau_think 0).
Writes one JSON document (stdout and --out) with the card's name and power limit read in the same run, before and
after, and per workload: both checks' verdicts, causes, repairs, bans, K15's lift steps and pairs lifted, both checks'
kernel time (CUDA events) and call time (every repeat after the warm-ups, and the medians), and, where the oracle runs
(the panel and the 10^6-op, 8-account, p_info 0 history), whether the device equals LW_SEARCH (commit_read included).

    python scripts/lifted_witness_bench.py --out /tmp/lifted_witness_bench.json
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
          "rounds", "repairs", "n_bans", "lifts", "n_lifted", "shards")


def causes(r) -> list:
    return sorted({abi.CAUSE_NAME[s["cause"]] or "none" for s in r["shards"]})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true", help="skip LW_SEARCH")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    loads = [("10^6", a.ops, n, p, 1, 0.0) for n in (8, 64) for p in (0.0, 0.02)] + [("C3", 10_000, 8, 0.02, 1, None)]
    loads += [("panel", 100_000, n, p, seed, 0.0) for n in (8, 64) for p in (0.0, 0.02) for seed in (1, 2)]
    doc = {"card": card(), "workloads": []}
    with native.Context(device=0) as ctx:
        for name, ops, n_acct, p_info, seed, tau in loads:
            kw = {} if tau is None else {"tau_think_ns": tau}
            h = synth.generate_ledger_lookups(synth.SynthSpec("bank", ops, 32, seed, p_info=p_info, n_accounts=n_acct,
                                                              final_reads=True, **kw))
            lw, lw_calls = timed(lambda: ctx.check_lifted_witness(h, witness=True), a.warmup, a.repeats)
            rw, rw_calls = timed(lambda: ctx.check_repaired_witness(h, witness=True), a.warmup, a.repeats)
            g, k = lw[-1], rw[-1]
            w = {"workload": name, "ops": ops, "accounts": n_acct, "p_info": p_info, "seed": seed,
                 "reads": g["n_reads"], "valid": g["valid"], "causes": causes(g), "repairs": g["repairs"],
                 "bans": g["n_bans"], "lifts": g["lifts"], "lifted": g["n_lifted"], "witness_rounds": g["rounds"],
                 "nodes": g["nodes"], "k14_valid": k["valid"], "k14_causes": causes(k), "k14_repairs": k["repairs"],
                 "k14_bans": k["n_bans"],
                 "median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in lw),
                 "median_seconds_call": statistics.median(lw_calls),
                 "k14_median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in rw),
                 "k14_median_seconds_call": statistics.median(rw_calls),
                 "seconds_kernel": [r["seconds_kernel"] for r in lw], "seconds_call": lw_calls,
                 "k14_seconds_kernel": [r["seconds_kernel"] for r in rw], "k14_seconds_call": rw_calls,
                 "repeats_equal": all({f: r[f] for f in FIELDS} == {f: g[f] for f in FIELDS} and
                                      np.array_equal(r["commit_read"], g["commit_read"]) for r in lw)}
            if not a.no_oracle and (name == "panel" or (name == "10^6" and n_acct == 8 and p_info == 0.0)):
                t0 = time.perf_counter()
                o = mono_oracle.check_lifted_witness(h)
                w["oracle_lw_search_seconds"] = time.perf_counter() - t0
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
