#!/usr/bin/env python3
"""WAV files in, MP3 files out: encode_wav_files against the host route it replaces.

Two arms on the same in-memory WAV files, alternated in one run, each timed with a host clock around a call that ends in a
device synchronise (parsing, PCM upload and byte read-back included):
  (a) numpy: WavHeader.readHeader per file, the data region de-interleaved with numpy on the host, encode_streams
  (b) wav:   encode_wav_files (raw data regions uploaded as they are, de-interleaved on the GPU by k_stage_wav)
Shapes: one C2-shaped stereo 44.1 kHz 128 kbps file of 10000 frames, 100 stereo 48 kHz 320 kbps files x 1000 frames (c3),
1000 mono 44.1 kHz 128 kbps files x 1000 frames (c4).  Arm (b)'s bytes must equal arm (a)'s.  k_stage_wav's own time comes
from torch.profiler (CUDA activities) in a separate, untimed pass.  The card's name and power limit are read in the same run.

  python tools/bench_wav.py --steps 5 --warmup 1 [--out bench_wav.json]
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

SHAPES = {  # name -> (channels, rate, kbps, files, frames per file, signal)
    "c2_1x10000_stereo44k": (2, 44100, 128, 1, 10000, "sweep"),
    "c3_100x1000_stereo48k": (2, 48000, 320, 100, 1000, "white"),
    "c4_1000x1000_mono44k": (1, 44100, 128, 1000, 1000, "octave"),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return None, None


def make_files(ch, sr, S, frames, kind):
    from synth import make_signal
    n = frames * 1152
    hdr = lambda nbytes: (b"RIFF" + (36 + nbytes).to_bytes(4, "little") + b"WAVEfmt " + (16).to_bytes(4, "little") +
                          np.array([1, ch], "<u2").tobytes() + np.array([sr, sr * ch * 2], "<u4").tobytes() +
                          np.array([ch * 2, 16], "<u2").tobytes() + b"data" + nbytes.to_bytes(4, "little"))
    files = []
    for s in range(S):
        l, r = make_signal(kind, n, sr, seed=1000 + s)
        x = np.stack([l, r], axis=1)[:, :ch]
        files.append(hdr(x.nbytes) + np.ascontiguousarray(x, dtype="<i2").tobytes())
    return files


def arm_numpy(M, files, kbps):
    lefts, rights, cfg = [], [], None
    for f in files:
        w = M.WavHeader.readHeader(f)
        v = np.frombuffer(f, dtype="<i2", count=w.dataLen // 2, offset=w.dataOffset)
        cfg = (w.channels, w.sampleRate)
        if w.channels == 2:
            lefts.append(np.ascontiguousarray(v[0::2]))
            rights.append(np.ascontiguousarray(v[1::2]))
        else:
            lefts.append(v)
    return M.encode_streams(cfg[0], cfg[1], kbps, lefts, rights if cfg[0] == 2 else None)


def arm_wav(M, files, kbps):
    mp3s, status = M.encode_wav_files(files, kbps)
    assert all(s == M.WAV_ENCODED for s in status)
    return mp3s


def stage_time_ms(M, files, kbps):
    """k_stage_wav's summed kernel time in one encode_wav_files call (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        arm_wav(M, files, kbps)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_stage_wav" in e.key)
    n = sum(e.count for e in prof.key_averages() if "k_stage_wav" in e.key)
    return us / 1000.0, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import lamejs_b200 as M
    name, limit = card()
    res = {"card": name, "power_limit": limit, "steps": a.steps, "warmup": a.warmup, "shapes": {}}
    for shape in a.shapes.split(","):
        ch, sr, kbps, S, frames, kind = SHAPES[shape]
        files = make_files(ch, sr, S, frames, kind)
        arms = {"numpy_deinterleave_encode_streams": arm_numpy, "encode_wav_files": arm_wav}
        ref = None
        for _ in range(a.warmup):
            for fn in arms.values():
                out = fn(M, files, kbps)
                ref = out if ref is None else ref
                assert out == ref, "arm bytes differ"
        times = {k: [] for k in arms}
        for _ in range(a.steps):
            for k, fn in arms.items():
                t0 = time.perf_counter()
                out = fn(M, files, kbps)                      # each call returns after its stream has drained
                times[k].append(time.perf_counter() - t0)
                assert out == ref, "arm bytes differ"
        audio_s = S * frames * 1152 / sr
        row = {"files": S, "frames_per_file": frames, "channels": ch, "samplerate": sr, "kbps": kbps,
               "wav_mb": round(sum(len(f) for f in files) / 1e6, 1), "bytes_equal": True}
        for k, ts in times.items():
            med = statistics.median(ts)
            row[k] = {"median_ms": round(med * 1e3, 2), "min_ms": round(min(ts) * 1e3, 2), "max_ms": round(max(ts) * 1e3, 2),
                      "audio_s_per_s": round(audio_s / med)}
        row["speedup_median"] = round(row["numpy_deinterleave_encode_streams"]["median_ms"] / row["encode_wav_files"]["median_ms"], 3)
        ms, nlaunch = stage_time_ms(M, files, kbps)
        row["k_stage_wav_ms"] = round(ms, 3)
        row["k_stage_wav_launches"] = nlaunch
        res["shapes"][shape] = row
        print(json.dumps({shape: row}), flush=True)
        del files
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
