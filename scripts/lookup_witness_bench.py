"""Time the lookup witness (K17) next to the class witness (K16).

Workloads: K16's six (scripts/class_witness_bench.py: the four 10^6-op ledger-lookups histories, 32 clients, tau_think
0, seed 1, one quiesced final read and lookup per client, 8 and 64 accounts x p_info 0 and 0.02; C3, 10,000 ops, 32
clients, seed 1, p_info 0.02; and the 10^5-op, 8-account, p_info 0.02, seed 2 history), plus two histories with
mid-run lookups (64 accounts, p_info 0.02, seed 1): 10^5 ops at p_lookup 0.01 and --ops ops at p_lookup 10^-4 (each
mid-run lookup returns every transfer committed before it, so the records grow with ops x lookups).  Writes one JSON
document (stdout and --out) with the card's name and power limit read in the same run, before and after, and per workload: both checks'
verdicts and causes, K17's lookup causes and lookups placed, both checks' kernel time (CUDA events) and call time
(every repeat after the warm-ups, and the medians).

    python scripts/lookup_witness_bench.py --out /tmp/lookup_witness_bench.json
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from jepsen_tigerbeetle_b200 import abi, native, synth  # noqa: E402
from serial_witness_bench import card, timed  # noqa: E402


def causes(r, field="cause") -> list:
    return sorted({abi.CAUSE_NAME[s[field]] or "none" for s in r["shards"]})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--ops", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    loads = [("10^6", a.ops, n, p, 1, 0.0, 0.0) for n in (8, 64) for p in (0.0, 0.02)]
    loads += [("C3", 10_000, 8, 0.02, 1, None, 0.0), ("10^5", 100_000, 8, 0.02, 2, 0.0, 0.0),
              ("mid-run lookups", 100_000, 64, 0.02, 1, 0.0, 0.01), ("mid-run lookups", a.ops, 64, 0.02, 1, 0.0, 1e-4)]
    doc = {"card": card(), "workloads": []}
    with native.Context(device=0) as ctx:
        for name, ops, n_acct, p_info, seed, tau, p_lookup in loads:
            kw = {} if tau is None else {"tau_think_ns": tau}
            h = synth.generate_ledger_lookups(synth.SynthSpec("bank", ops, 32, seed, p_info=p_info, n_accounts=n_acct,
                                                              final_reads=True, **kw), p_lookup=p_lookup)
            lk, lk_calls = timed(lambda: ctx.check_lookup_witness(h, witness=True), a.warmup, a.repeats)
            cw, cw_calls = timed(lambda: ctx.check_class_witness(h, witness=True), a.warmup, a.repeats)
            g, k = lk[-1], cw[-1]
            w = {"workload": name, "ops": ops, "accounts": n_acct, "p_info": p_info, "p_lookup": p_lookup,
                 "seed": seed, "reads": g["n_reads"], "lookups": int(abi.n_ok_lookups(h)), "valid": g["valid"],
                 "causes": causes(g), "lookup_causes": causes(g, "lookup_cause"), "placed": g["n_lookups_placed"],
                 "k16_valid": k["valid"], "k16_causes": causes(k),
                 "median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in lk),
                 "median_seconds_call": statistics.median(lk_calls),
                 "k16_median_seconds_kernel": statistics.median(r["seconds_kernel"] for r in cw),
                 "k16_median_seconds_call": statistics.median(cw_calls),
                 "seconds_kernel": [r["seconds_kernel"] for r in lk], "seconds_call": lk_calls,
                 "k16_seconds_kernel": [r["seconds_kernel"] for r in cw], "k16_seconds_call": cw_calls}
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
