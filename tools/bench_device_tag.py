#!/usr/bin/env python3
"""Cost of the tag (and of ReplayGain) on the device-resident whole-stream path.

For C2 (one stereo 44.1 kHz 128 kbps sweep of 10000 frames) and a c3-shaped batch (stereo 48 kHz 320 kbps, 100 white-noise
streams of 1000 frames), with the PCM on the device as Int16 and as Float32 (the same samples / 32768: Web Audio scale, what a
Float32 caller feeds), four arms are timed alternately in one run, each with a host clock around a whole call that ends in a
device synchronise:
  device              encode_streams_device (untagged)
  device_tag          encode_streams_device_tagged
  device_tag_rg       encode_streams_device_tagged(find_replay_gain=True)
  host_copy_tag_rg    what a caller whose PCM is on the device did before the tagged device path existed: copy the PCM to
                      the host, then encode_streams_replaygain (mp3b200_encode_streams_tagged_ex with MP3B200_REPLAYGAIN),
                      which uploads it again and returns the files in host memory
The files of the two tagged device arms are checked against the host path's.  Prints the device name and power limit with
the numbers.

  python tools/bench_device_tag.py --steps 10 --warmup 3
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

ARMS = ("device", "device_tag", "device_tag_rg", "host_copy_tag_rg")


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
        ns = [len(l) for l, _ in sig]
        pcm = np.concatenate([np.concatenate([l, r]) for l, r in sig])
        pcm_off = np.concatenate([[0], np.cumsum([2 * n for n in ns])[:-1]])
        nb = [M.stream_bytes(ch, sr, kb, n) for n in ns]
        tfs = M.lametag_size(ch, sr, kb)
        out_off = np.concatenate([[0], np.cumsum(nb)[:-1]])
        tag_off = np.concatenate([[0], np.cumsum([b + tfs for b in nb])[:-1]])
        for fmt in ("int16", "float32"):
            f32 = fmt == "float32"
            d_pcm = torch.from_numpy(pcm).cuda()
            if f32:
                d_pcm = d_pcm.float() / 32768.0
            d_out = torch.zeros(sum(nb) + 8, dtype=torch.uint8, device="cuda")
            d_tag = torch.zeros(sum(nb) + tfs * len(nb) + 8, dtype=torch.uint8, device="cuda")
            files = {}

            def run(arm):
                if arm == "device":
                    M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), pcm_off, ns, d_out.data_ptr(), out_off, float32=f32)
                elif arm in ("device_tag", "device_tag_rg"):
                    M.encode_streams_device_tagged(ch, sr, kb, d_pcm.data_ptr(), pcm_off, ns, d_tag.data_ptr(), tag_off, float32=f32,
                                                   find_replay_gain=(arm == "device_tag_rg"))
                else:
                    h = d_pcm.cpu().numpy()
                    lefts = [h[o:o + n] for o, n in zip(pcm_off, ns)]
                    rights = [h[o + n:o + 2 * n] for o, n in zip(pcm_off, ns)]
                    files[arm] = M.encode_streams_replaygain(ch, sr, kb, lefts, rights)[0]

            for _ in range(a.warmup):
                for arm in ARMS:
                    run(arm)
            ms = {arm: [] for arm in ARMS}
            for i in range(a.steps):
                for arm in (ARMS if i % 2 == 0 else ARMS[::-1]):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    run(arm)
                    torch.cuda.synchronize()
                    ms[arm].append((time.perf_counter() - t0) * 1e3)
            run("device_tag_rg")
            t = d_tag.cpu().numpy().tobytes()
            same = [t[o:o + b + tfs] for o, b in zip(tag_off, nb)] == files["host_copy_tag_rg"]
            med = {arm: statistics.median(v) for arm, v in ms.items()}
            res["workloads"]["%s_%s" % (name, fmt)] = {"streams": len(ns), "samples_per_channel": ns[0], "call_ms_median": med,
                                                       "call_ms": ms, "files_equal_host": same}
            print(name, fmt, json.dumps(med), "files_equal_host", same, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
