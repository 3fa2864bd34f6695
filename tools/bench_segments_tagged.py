#!/usr/bin/env python3
"""Cost of the pieces of a segmented finished file on one GPU, for the C2-shaped stream (one stereo 44.1 kHz 128 kbps sweep
of 10000 frames, device-resident Int16 rows).  Arms, alternated in one run (host clock around calls that end in a device
synchronise):
  tagged_rg        encode_streams_device_tagged(find_replay_gain=True): the whole-stream finished file
  analysis         replay_gain_streams_device alone (no encoder kernel)
  finish           finish_tags_device alone, on the untagged audio placed behind the tag's room
  segments_1 / _8  sharding.encode_stream_segments_tagged_local with ReplayGain at nseg 1 and 8 (one GPU, ranges in turn,
                   host rows and host bytes as the handle API takes them)
Prints one JSON line with the median and min of each arm in ms, the device name and its power limit.

  python tools/bench_segments_tagged.py --steps 5 --warmup 1
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
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--frames", type=int, default=10000)
    a = ap.parse_args()
    import torch
    import lamejs_b200 as M
    from lamejs_b200 import sharding
    from synth import make_signal

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    ch, sr, kb = 2, 44100, 128
    l, r = make_signal("sweep", a.frames * 1152, sr, seed=1)
    n = len(l)
    d_pcm = torch.from_numpy(np.concatenate([l, r])).cuda()
    tfs = M.lametag_size(ch, sr, kb)
    nbytes = M.stream_bytes(ch, sr, kb, n)
    d_out = torch.zeros(nbytes + tfs, dtype=torch.uint8, device="cuda")
    d_audio = torch.zeros(nbytes + tfs, dtype=torch.uint8, device="cuda")
    M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [n], d_audio.data_ptr(), [tfs])
    title, _ = M.replay_gain_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [n])

    def tagged_rg():
        M.encode_streams_device_tagged(ch, sr, kb, d_pcm.data_ptr(), [0], [n], d_out.data_ptr(), [0], find_replay_gain=True)

    def analysis():
        M.replay_gain_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [n])

    def finish():
        M.finish_tags_device(ch, sr, kb, d_audio.data_ptr(), [0], [n], title)

    def segments(nseg):
        return lambda: sharding.encode_stream_segments_tagged_local(ch, sr, kb, l, r, nseg, 8, find_replay_gain=True)

    arms = {"tagged_rg": tagged_rg, "analysis": analysis, "finish": finish, "segments_1": segments(1), "segments_8": segments(8)}
    # the arms make the same file: the check that what is timed is what the tests pin
    tagged_rg()
    seg = sharding.encode_stream_segments_tagged_local(ch, sr, kb, l, r, 8, 8, find_replay_gain=True)
    finish()
    same = seg[0] == d_out.cpu().numpy().tobytes() == d_audio.cpu().numpy().tobytes()
    times = {k: [] for k in arms}
    for step in range(a.warmup + a.steps):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if step >= a.warmup:
                times[k].append(1e3 * (time.perf_counter() - t0))
    print(json.dumps({"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "frames": a.frames,
                      "files_equal": bool(same), "title_db": title[0],
                      "ms": {k: {"median": statistics.median(v), "min": min(v)} for k, v in times.items()}}))


if __name__ == "__main__":
    main()
