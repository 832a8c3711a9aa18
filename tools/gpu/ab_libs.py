#!/usr/bin/env python3
"""A/B timing of libnmsm builds: runs bench.py against each build in turn (NMSM_LIB), alternating the builds round by
round so that drift of the card or of its neighbours hits all of them alike, and prints the median and the spread of
each metric per build.

  python tools/gpu/ab_libs.py [--rounds 3] [--configs] LABEL=LIB[,VAR=VALUE...] ... [-- bench.py arguments]

LIB is a path to a libnmsm.so; VAR=VALUE pairs are extra environment for that build's runs (e.g. NMSM_L=56 to plan a
build's segments for another occupancy).  Every run's JSON line goes to stdout as it finishes, then one summary line per
build; the card's name, power limit and maximum SM clock are read first, because they are part of every number."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def metrics(line, configs):
    """The numbers compared between builds, from one bench.py JSON line."""
    if configs:
        return {"config%d_ms_device" % r["config"]: r["ms_device"] for r in line["configs"] if "ms_device" in r}
    m = {"ms_per_step": line["ms_per_step"], "device_ms_per_step": line["device_ms_per_step"]}
    roof = line.get("roofline") or {}
    if roof.get("kernel_ms_breakdown_linear"):
        m["accumulate_ms_linear"] = roof["kernel_ms_breakdown_linear"].get("accumulate")
        m["accumulate_frac_of_modmul_peak"] = roof.get("frac")
    for key in ("fixed_base", "any_point"):
        if line.get(key):
            m[key + "_ms_per_step"] = line[key]["ms_per_step"]
    return m


def main():
    argv = sys.argv[1:]
    bench_args = []
    if "--" in argv:
        i = argv.index("--")
        argv, bench_args = argv[:i], argv[i + 1:]
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", action="store_true", help="time bench.py --configs instead of the headline")
    ap.add_argument("builds", nargs="+", metavar="LABEL=LIB[,VAR=VALUE...]")
    args = ap.parse_args(argv)
    builds = []
    for spec in args.builds:
        label, rest = spec.split("=", 1)
        path, *env = rest.split(",")
        builds.append((label, os.path.abspath(path), dict(e.split("=", 1) for e in env)))
    print(json.dumps({"card": card(), "bench_args": bench_args, "rounds": args.rounds}), flush=True)
    runs = {label: [] for label, _, _ in builds}
    for rnd in range(args.rounds):
        for label, path, extra in builds:
            env = dict(os.environ, NMSM_LIB=path, **extra)
            cmd = [sys.executable, os.path.join(ROOT, "bench.py")] + (["--configs"] if args.configs else []) + bench_args
            p = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
            out = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
            if p.returncode != 0 or not out:
                print(json.dumps({"build": label, "round": rnd, "rc": p.returncode, "stderr": p.stderr[-2000:]}), flush=True)
                continue
            m = metrics(json.loads(out[-1]), args.configs)
            runs[label].append(m)
            print(json.dumps({"build": label, "round": rnd, **m}), flush=True)
    for label, _, extra in builds:
        rs = runs[label]
        summary = {"build": label, "env": extra, "runs": len(rs)}
        for k in (rs[0] if rs else {}):
            v = [r[k] for r in rs if r.get(k) is not None]
            if v:
                med = statistics.median(v)
                summary[k] = {"median": med, "min": min(v), "max": max(v),
                              "spread_pct": 100.0 * (max(v) - min(v)) / med if med else None}
        print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
