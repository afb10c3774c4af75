"""A/B of library builds on the flagship benchmark: runs `bench.py` alternately for each build, several rounds, each in a
fresh process (a build other than the in-tree one is selected with JTB_LIB_PATH), dumps each build's outputs and
compares them file by file.

    python scripts/ab_bench.py --out DIR [--rounds 3] [--invalid] NAME=LIB_OR_DEFAULT[:ENV=V,...] ...

`default` as the library means the in-tree build.  Prints one JSON line per run, then a summary per build (median,
min and max of `value`, kernel time per step, probes, tile-filter drops) and whether the dumped arrays are identical;
everything is also written to DIR/ab_bench.json."""
import argparse
import glob
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def parse_build(s):
    name, rest = s.split("=", 1)
    lib, _, envs = rest.partition(":")
    env = {}
    if lib != "default":
        env["JTB_LIB_PATH"] = os.path.abspath(lib)
    if envs:
        env.update(kv.split("=", 1) for kv in envs.split(","))
    return name, env


def run(name, envx, args, tag, invalid):
    out = os.path.join(args.out, f"dump_{name}_{tag}")
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps), "--warmup",
           str(args.warmup), "--dump-outputs", out]
    if invalid:
        cmd += ["--invalid", "--no-full-run", "--no-sharded"]
    if args.no_cpu_baseline:
        cmd.append("--no-cpu-baseline")
    env = dict(os.environ)
    env.update(envx)
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=3000)
    line = None
    for ln in r.stdout.splitlines():
        if ln.startswith("{"):
            line = json.loads(ln)
    if line is None:
        return {"error": r.stderr[-3000:]}, out
    return line, out


def same_dumps(a, b):
    fa = sorted(os.path.basename(f) for f in glob.glob(os.path.join(a, "*.npy")))
    fb = sorted(os.path.basename(f) for f in glob.glob(os.path.join(b, "*.npy")))
    return fa == fb and len(fa) > 0 and all(np.array_equal(np.load(os.path.join(a, f)), np.load(os.path.join(b, f)))
                                            for f in fa)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--invalid", action="store_true", help="also one --invalid run per build")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("builds", nargs="+")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    builds = [parse_build(b) for b in args.builds]
    res = {name: [] for name, _ in builds}
    dumps = {name: [] for name, _ in builds}
    for rnd in range(args.rounds):
        for name, env in builds:
            line, d = run(name, env, args, f"r{rnd}", False)
            res[name].append(line)
            dumps[name].append(d)
            short = {k: line.get(k) for k in ("value", "time_to_verdict_kernel_s", "configs_per_step", "probes_per_step",
                                              "verdict", "error")}
            print(name, rnd, json.dumps(short), flush=True)
    inval = {}
    if args.invalid:
        for name, env in builds:
            line, d = run(name, env, args, "invalid", True)
            inval[name] = {k: line.get(k) for k in ("value", "time_to_verdict_kernel_s", "configs_per_step",
                                                    "probes_per_step", "verdict", "error")}
            dumps[name].append(d)
            print(name, "invalid", json.dumps(inval[name]), flush=True)
    ref = builds[0][0]
    summary = {}
    for name, _ in builds:
        ok = [x for x in res[name] if "value" in x]
        vals = [x["value"] for x in ok]
        summary[name] = {
            "value_median": statistics.median(vals) if vals else None,
            "value_min": min(vals) if vals else None, "value_max": max(vals) if vals else None,
            "kernel_s_per_step": [x["time_to_verdict_kernel_s"] for x in ok],
            "probes_per_step": [x["probes_per_step"] for x in ok],
            "configs_per_step": sorted({x["configs_per_step"] for x in ok}),
            "verdicts": sorted({x["verdict"] for x in ok}),
            "v2v_s": [x.get("verdict_to_verdict", {}).get("time_to_verdict_s") for x in ok],
            "eager_s": [x.get("product_default_eager_reads", {}).get("time_to_verdict_s") for x in ok],
            "sharded": [x.get("sharded") for x in ok],
            "clocks": ok[-1].get("clocks") if ok else None,
            "dumps_identical_to_" + ref: all(same_dumps(a, b) for a, b in zip(dumps[ref], dumps[name])),
            "invalid": inval.get(name),
        }
    print(json.dumps(summary, indent=1))
    json.dump({"runs": res, "summary": summary}, open(os.path.join(args.out, "ab_bench.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
