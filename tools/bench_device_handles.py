#!/usr/bin/env python3
"""Cost of feeding streaming handles from device memory (mp3b200_encode_batch_device / mp3b200_encode_device) against
copying the samples to the host first.

Two workloads, each with two arms timed alternately in one run, a host clock around each call (the calls return the bytes in
host memory, so each ends with the device drained):
  live   512 mono handles at a native 24 kHz configuration; every round torch makes a 100 ms Float32 chunk per handle on the
         GPU (2400 samples), for 50 rounds.  (a) host: encode_batch of t.cpu()   (b) device: encode_batch of t
  whole  C2 (stereo 44.1 kHz 128 kbps sweep, 10 001 frames, Int16) through one fresh handle's encodeBuffer + flush,
         (a) from host memory   (b) from a CUDA tensor
Reports the median ms per round / per file of each arm and whether both arms gave identical bytes, with the device name
and power limit.  --profile DIR also writes a torch.profiler summary of one device round of each workload into DIR.

  python tools/bench_device_handles.py --rounds 50 --steps 5 --warmup 2
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


def live_kbps(M):
    for kb in (64, 48, 56, 40, 32, 80, 96):
        if M.out_samplerate(1, 24000, kb) == 24000:
            return kb
    raise SystemExit("no native 24 kHz mono configuration")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--handles", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--steps", type=int, default=5, help="whole-file runs per arm")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", default=None, metavar="DIR")
    a = ap.parse_args()
    import torch
    import lamejs_b200 as M
    from synth import make_signal

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}

    # ---- live: 512 handles, 100 ms Float32 chunks made on the GPU ----
    kb, S, n = live_kbps(M), a.handles, 2400
    encs = {arm: [M.Mp3Encoder(1, 24000, kb) for _ in range(S)] for arm in ("host", "device")}
    f = torch.linspace(200.0, 3000.0, S, device="cuda", dtype=torch.float64)[:, None]
    k = torch.arange(n, device="cuda", dtype=torch.float64)[None, :]

    def chunk(r):
        t = (r * n + k) / 24000.0
        return (0.4 * torch.sin(2 * np.pi * f * t) + 0.05 * torch.sin(2 * np.pi * 7.0 * f * t)).float()

    def live_round(arm, t):
        rows = list(t.cpu()) if arm == "host" else list(t)
        return M.encode_batch(encs[arm], rows)

    ms = {"host": [], "device": []}
    same = True
    for r in range(a.warmup + a.rounds):
        t = chunk(r)
        torch.cuda.synchronize()
        outs = {}
        for arm in (("host", "device") if r % 2 == 0 else ("device", "host")):
            t0 = time.perf_counter()
            outs[arm] = live_round(arm, t)
            dt = (time.perf_counter() - t0) * 1e3
            if r >= a.warmup:
                ms[arm].append(dt)
        same = same and outs["host"] == outs["device"]
    same = same and M.flush_batch(encs["host"]) == M.flush_batch(encs["device"])
    res["live"] = {"handles": S, "kbps": kb, "samples_per_round": n, "rounds": a.rounds,
                   "round_ms_median": {arm: statistics.median(v) for arm, v in ms.items()}, "bytes_equal": same}
    print("live", json.dumps(res["live"]), flush=True)

    # ---- whole file: C2 through one handle ----
    l, rgt = make_signal("sweep", 10000 * 1152, 44100, seed=1)
    dl, dr = torch.from_numpy(l).cuda(), torch.from_numpy(rgt).cuda()

    def whole(arm):
        e = M.Mp3Encoder(2, 44100, 128)
        b = (e.encodeBuffer(l, rgt) if arm == "host" else e.encodeBuffer(dl, dr)) + e.flush()
        e.close()
        return b

    ms = {"host": [], "device": []}
    files = {}
    for i in range(a.warmup + a.steps):
        for arm in (("host", "device") if i % 2 == 0 else ("device", "host")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            files[arm] = whole(arm)
            dt = (time.perf_counter() - t0) * 1e3
            if i >= a.warmup:
                ms[arm].append(dt)
    res["whole"] = {"frames": 10001, "file_ms_median": {arm: statistics.median(v) for arm, v in ms.items()},
                    "bytes_equal": files["host"] == files["device"]}
    print("whole", json.dumps(res["whole"]), flush=True)

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        for name, fn in (("live", lambda: live_round("device", chunk(0))), ("whole", lambda: whole("device"))):
            fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
                fn()
                torch.cuda.synchronize()
            tab = p.key_averages().table(sort_by="cuda_time_total", row_limit=25)
            with open(os.path.join(a.profile, "profile_device_handles_%s.txt" % name), "w") as fh:
                fh.write(tab)
            print(tab, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
