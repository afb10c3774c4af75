"""Time the class witness (K16) next to the lifted serial witness (K15), and compare it with the CW_SEARCH CPU oracle.

Workloads: K15's five (the four 10^6-op ledger-lookups histories, 32 clients, tau_think 0, seed 1, one quiesced final
read and lookup per client, 8 and 64 accounts x p_info 0 and 0.02; and C3, 10,000 ops, 32 clients, seed 1, p_info
0.02) and the 10^5-op, 8-account, p_info 0.02, seed 2 panel history, the one K15 leaves no-witness.  Writes one JSON
document (stdout and --out) with the card's name and power limit read in the same run, before and after, and per
workload: both checks' verdicts and causes, K16's class cause, class rounds and members handed out, both checks'
kernel time (CUDA events) and call time (every repeat after the warm-ups, and the medians), and, where the oracle runs
(the 10^5-op history and the 10^6-op, 8-account, p_info 0.02 history), whether the device equals CW_SEARCH
(commit_read included).

    python scripts/class_witness_bench.py --out /tmp/class_witness_bench.json
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
          "rounds", "repairs", "n_bans", "lifts", "n_lifted", "class_rounds", "n_handed", "shards")


def causes(r, field="cause") -> list:
    return sorted({abi.CAUSE_NAME[s[field]] or "none" for s in r["shards"]})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-oracle", action="store_true", help="skip CW_SEARCH")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    loads = [("10^6", a.ops, n, p, 1, 0.0) for n in (8, 64) for p in (0.0, 0.02)] + [("C3", 10_000, 8, 0.02, 1, None)]
    loads += [("10^5", 100_000, 8, 0.02, 2, 0.0)]
    doc = {"card": card(), "workloads": []}
    with native.Context(device=0) as ctx:
        for name, ops, n_acct, p_info, seed, tau in loads:
            kw = {} if tau is None else {"tau_think_ns": tau}
            h = synth.generate_ledger_lookups(synth.SynthSpec("bank", ops, 32, seed, p_info=p_info, n_accounts=n_acct,
                                                              final_reads=True, **kw))
            cw, cw_calls = timed(lambda: ctx.check_class_witness(h, witness=True), a.warmup, a.repeats)
            lw, lw_calls = timed(lambda: ctx.check_lifted_witness(h, witness=True), a.warmup, a.repeats)
            g, k = cw[-1], lw[-1]
            w = {"workload": name, "ops": ops, "accounts": n_acct, "p_info": p_info, "seed": seed,
                 "reads": g["n_reads"], "valid": g["valid"], "causes": causes(g),
                 "class_causes": causes(g, "class_cause"), "class_rounds": g["class_rounds"],
                 "handed": g["n_handed"], "nodes": g["nodes"], "k15_valid": k["valid"], "k15_causes": causes(k),
                 "median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in cw),
                 "median_seconds_call": statistics.median(cw_calls),
                 "k15_median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in lw),
                 "k15_median_seconds_call": statistics.median(lw_calls),
                 "seconds_kernel": [r["seconds_kernel"] for r in cw], "seconds_call": cw_calls,
                 "k15_seconds_kernel": [r["seconds_kernel"] for r in lw], "k15_seconds_call": lw_calls,
                 "repeats_equal": all({f: r[f] for f in FIELDS} == {f: g[f] for f in FIELDS} and
                                      np.array_equal(r["commit_read"], g["commit_read"]) for r in cw)}
            if not a.no_oracle and (name == "10^5" or (name == "10^6" and n_acct == 8 and p_info == 0.02)):
                t0 = time.perf_counter()
                o = mono_oracle.check_class_witness(h)
                w["oracle_cw_search_seconds"] = time.perf_counter() - t0
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
