#!/usr/bin/env python3
"""Cost of ReplayGain analysis (MP3B200_REPLAYGAIN) on the tagged whole-stream path.

For C2 (one stereo 44.1 kHz 128 kbps sweep of 10000 frames) and a c3-shaped batch (stereo 48 kHz 320 kbps, 100 white-noise
streams of 1000 frames) it times encode_streams_tagged with the analysis off and on, alternating the two in one run
(host clock around calls that end in a device synchronise, PCM upload and byte read-back included), and reports the
analysis's own CUDA-event time, its repair passes and the chunks it ran again (mp3b200_debug_replaygain on the first
stream), with the device name and power limit.

  python tools/bench_replaygain.py --steps 10 --warmup 3
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import lamejs_b200 as M
    from synth import make_signal

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "workloads": {}}
    work = {
        "c2": (2, 44100, 128, [make_signal("sweep", 10000 * 1152, 44100, seed=1)]),
        "c3": (2, 48000, 320, [make_signal("white", 1000 * 1152, 48000, seed=s) for s in range(100)]),
    }
    for name, (ch, sr, kb, sig) in work.items():
        lefts, rights = [s[0] for s in sig], [s[1] for s in sig]

        def off():
            M.encode_streams_tagged(ch, sr, kb, lefts, rights)

        def on():
            M.encode_streams_replaygain(ch, sr, kb, lefts, rights)

        for _ in range(a.warmup):
            off()
            on()
        t_off, t_on = [], []
        for i in range(a.steps):
            for f, acc in ((off, t_off), (on, t_on)) if i % 2 == 0 else ((on, t_on), (off, t_off)):
                t0 = time.perf_counter()
                f()
                acc.append((time.perf_counter() - t0) * 1e3)
        d = M.debug_replaygain(ch, sr, kb, lefts[0], rights[0])
        res["workloads"][name] = {
            "streams": len(lefts), "samples_per_channel": len(lefts[0]),
            "rg_off_ms_median": statistics.median(t_off), "rg_on_ms_median": statistics.median(t_on),
            "rg_off_ms": t_off, "rg_on_ms": t_on,
            "rg_kernels_ms_first_stream": d["ms"], "repair_passes": d["passes"], "chunks_rerun": d["reruns"],
            "windows_first_stream": int(len(d["idx"])),
        }
        print(name, json.dumps(res["workloads"][name]["rg_off_ms_median"]), json.dumps(res["workloads"][name]["rg_on_ms_median"]),
              d["ms"], d["passes"], d["reruns"], flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
