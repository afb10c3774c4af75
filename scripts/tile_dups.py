"""Where the duplicates of a level are, on the CPU: the bench headline history (bank, 10k ops, 32 clients, seed 1,
tau_think 0, Knossos-exact space) walked level by level (tests/hostwalk_dups.py), printing for every level of at least
--min-width parents the children generated, the new configurations, and the children that repeat a key generated
from the same block of W consecutive parents — what a tile filter over tiles of W parents drops.

    python scripts/tile_dups.py [--max-configs 80000000] [--windows 32,256,2048] [--min-width 1000000]

The walk is single-threaded and keeps a level in host memory: --max-configs 200000000 (levels up to 22.8 M parents)
took about 15 minutes on one core.  The last level shown is cut short by the budget."""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import hostwalk_dups  # noqa: E402
from jepsen_tigerbeetle_b200 import history as H, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-configs", type=int, default=80_000_000)
    ap.add_argument("--windows", default="32,256,2048")
    ap.add_argument("--min-width", type=int, default=1_000_000)
    ap.add_argument("--ops", type=int, default=10000)
    args = ap.parse_args()
    windows = tuple(int(w) for w in args.windows.split(","))
    h = synth.generate(synth.SynthSpec("bank", args.ops, 32, 1, tau_think_ns=0.0, stale_read=False))
    m = H.make_model(H.MODEL_BANK, accounts=range(1, 9))
    t = time.time()
    r = hostwalk_dups.walk_dups(h, m, windows=windows, eager_reads=False, max_configs=args.max_configs)
    print(f"# {r['configs']:,} configurations, {r['levels']} levels, verdict {r['valid']} "
          f"(0 valid, 1 unknown = budget), {time.time() - t:.0f} s")
    print("| level | parents | children probed | new | " + " | ".join(f"dup. within {w} parents" for w in windows) + " |")
    print("|---|---|---|---|" + "---|" * len(windows))
    tot = {"children": 0, "new": 0, **{w: 0 for w in windows}}
    for lv, row in enumerate(r["rows"]):
        if row["parents"] < args.min_width:
            continue
        c = row["children"]
        tot["children"] += c
        tot["new"] += row["new"]
        cells = []
        for w in windows:
            tot[w] += row["dups"][w]
            cells.append(f"{row['dups'][w] / 1e6:.2f} M ({100 * row['dups'][w] / max(c, 1):.0f} %)")
        print(f"| {lv} | {row['parents'] / 1e6:.2f} M | {c / 1e6:.2f} M ({c / row['parents']:.1f} per parent) | "
              f"{row['new'] / 1e6:.2f} M | " + " | ".join(cells) + " |")
    if tot["children"]:
        c = tot["children"]
        print(f"# levels shown: {c:,} children, {tot['new']:,} new; duplicates within W: " +
              ", ".join(f"W={w}: {100 * tot[w] / c:.1f} % of children, {100 * tot[w] / max(c - tot['new'], 1):.1f} % of all "
                        f"duplicates, window probes per new configuration {(c - tot[w]) / max(tot['new'], 1):.2f}"
                        for w in windows))


if __name__ == "__main__":
    main()
