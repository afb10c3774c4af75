"""Throughput of the search kernel vs number of persistent CTAs (occupancy scaling experiment)."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from jepsen_tigerbeetle_b200 import native, synth, history as H
h = synth.generate(synth.SynthSpec("bank", 10000, 32, 1, tau_think_ns=5e6, stale_read=True))
m = H.make_model(H.MODEL_BANK, accounts=range(1, 9))
for ctas in (66, 132, 264, 396, 528):   # multiples of the H100's 132 SMs
    ctx = native.Context(device=0, search_ctas=ctas)
    for _ in range(2):
        r = ctx.check_linearizable(h, m)
    print(ctas, "ctas:", round(r["seconds_kernel"], 4), "s", round(r["configs"] / r["seconds_kernel"] / 1e6), "Mcfg/s", flush=True)
    ctx.close()
