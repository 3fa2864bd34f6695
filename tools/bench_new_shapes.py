#!/usr/bin/env python3
"""The cost of a launch shape a thread has not seen: one C2-length call (stereo 44.1 kHz 128 kbps, a 10 000-frame sine
sweep) per new length, each length called once, so that every call captures and instantiates its fixed-point loop graph.
Host time is the wall time of the synchronous call (it returns with the bytes on the device); device time is the
pipeline's CUDA-event total (timing slot 6).  The builds take turns, one process per build and round.

  python tools/bench_new_shapes.py --rounds 2 --shapes 20 name=LIB.so [name=LIB.so ...]

Prints one JSON line per build: medians in ms per call, and the card and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = (2, 44100, 128)


def worker(shapes):
    import numpy as np
    import torch

    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import lamejs_b200 as M
    from synth import sweep

    base = 10000 * 1152
    l, r = sweep(base + 1152 * (shapes + 2), 44100)
    pcm = torch.from_numpy(np.concatenate([l, r])).cuda()
    out = torch.zeros(M.stream_bytes(*CFG, len(l)) + 8, dtype=torch.uint8, device="cuda")

    def call(n):
        d = torch.from_numpy(np.concatenate([l[:n], r[:n]])).cuda() if n != len(l) else pcm
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tm = M.encode_streams_device(*CFG, d.data_ptr(), [0], [n], out.data_ptr(), [0])
        return (time.perf_counter() - t0) * 1e3, float(tm[6])

    for _ in range(3):                       # modules, tables and the workspace at its largest
        call(len(l))
    res = [call(base + 1152 * k + 17) for k in range(shapes)]
    warm = [call(base + 17) for _ in range(5)]   # the first shape again: its graph is cached
    p = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    print(json.dumps({"new_host_ms": [h for h, _ in res], "new_device_ms": [d for _, d in res],
                      "warm_host_ms": [h for h, _ in warm], "warm_device_ms": [d for _, d in warm],
                      "gpu": p.name, "power_limit": q.stdout.strip()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--shapes", type=int, default=20)
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("builds", nargs="*", help="name=path of a libmp3b200 build")
    args = ap.parse_args()
    if args.worker:
        return worker(args.shapes)
    acc = {}
    for _ in range(args.rounds):
        for name, lib in (b.split("=", 1) for b in args.builds):
            env = dict(os.environ, MP3B200_LIB=os.path.abspath(lib))
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--shapes", str(args.shapes)], env=env,
                               capture_output=True, text=True)
            if p.returncode != 0:
                sys.exit(p.stdout[-2000:] + p.stderr[-4000:])
            r = json.loads(p.stdout.strip().splitlines()[-1])
            a = acc.setdefault(name, {"gpu": r["gpu"], "power_limit": r["power_limit"]})
            for k, v in r.items():
                if k.endswith("_ms"):
                    a.setdefault(k, []).extend(v)
    for name, a in acc.items():
        print(json.dumps(dict({"build": name, "gpu": a["gpu"], "power_limit": a["power_limit"]},
                              **{k + "_median": round(statistics.median(v), 3) for k, v in a.items() if k.endswith("_ms")})))


if __name__ == "__main__":
    main()
