#!/usr/bin/env python3
"""A/B timing of library builds with the unchanged bench.py: the builds take turns, run after run, so that a drift of the
shared host or of the card's clock lands on all of them alike.

  python tools/bench_ab.py --runs 5 --out DIR name=LIB.so [name=LIB.so ...] -- --config c2 --steps 20 --warmup 5

Every run is `bench.py <args after -->` with MP3B200_LIB naming the build.  Prints, per build, the median and the min-max
spread of ms_per_step and of k_q_outer's per-step time, and the card, power limit and SM clock bench.py read; writes every
JSON line to DIR/bench_ab.jsonl."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    argv = sys.argv[1:]
    bench_args = argv[argv.index("--") + 1:] if "--" in argv else []
    argv = argv[:argv.index("--")] if "--" in argv else argv
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", required=True)
    ap.add_argument("builds", nargs="+", help="name=path of a libmp3b200 build")
    args = ap.parse_args(argv)
    builds = [b.split("=", 1) for b in args.builds]
    os.makedirs(args.out, exist_ok=True)
    res = {n: [] for n, _ in builds}
    with open(os.path.join(args.out, "bench_ab.jsonl"), "a") as log:
        for r in range(args.runs):
            for name, lib in builds:
                env = dict(os.environ, MP3B200_LIB=os.path.abspath(lib))
                p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + bench_args, env=env, cwd=ROOT,
                                   capture_output=True, text=True)
                lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
                if p.returncode != 0 or not lines:
                    sys.stderr.write(p.stdout[-2000:] + p.stderr[-4000:])
                    raise SystemExit("bench.py failed for %s (exit %d)" % (name, p.returncode))
                j = json.loads(lines[-1])
                log.write(json.dumps({"build": name, "run": r, "bench": j}) + "\n")
                log.flush()
                res[name].append(j)
                print("run %d %-10s ms_per_step %.4f  k_q_outer %.4f" % (
                    r, name, j["ms_per_step"], j["kernels"]["quantizer"]["by_kernel_ms"]["k_q_outer"]), flush=True)
    print()
    for name, js in res.items():
        st = [j["ms_per_step"] for j in js]
        ko = [j["kernels"]["quantizer"]["by_kernel_ms"]["k_q_outer"] for j in js]
        c = js[-1].get("clocks") or {}
        print("%-10s ms_per_step median %.4f (min %.4f max %.4f)  k_q_outer median %.4f (min %.4f max %.4f)  [%s, %s W, SM %s MHz]" % (
            name, statistics.median(st), min(st), max(st), statistics.median(ko), min(ko), max(ko), js[-1].get("device"),
            c.get("power_limit_w"), c.get("sm_mhz")))


if __name__ == "__main__":
    main()
