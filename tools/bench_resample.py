"""What resampling costs: 48 kHz -> 24 kHz stereo 64 kbps (new Mp3Encoder(2, 48000, 64)) against the native 24 kHz stereo
64 kbps encode of the same output frames, device-resident, in one process, the two alternating step by step.

usage: python tools/bench_resample.py [--steps K] [--warmup W]      (one H100)
Prints one JSON line: the card's name and power limit, and per case and path the median step time (host clock around the
synchronising call), the resampler's kernel time (CUDA events, timing slot 14) and audio seconds encoded per second."""
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
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    import lamejs_b200 as M
    from synth import make_signal

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    ch, kb = 2, 64
    cases = {"1x10001_frames": (1, 10001), "256x1000_frames": (256, 1000)}
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "steps": args.steps, "warmup": args.warmup,
           "config": "2ch 64 kbps, 48000 -> 24000 Hz resampled vs 24000 Hz native"}
    for name, (S, frames) in cases.items():
        n_out = frames * 576 - 2000                     # the shortest native input that makes `frames` frames
        while M.stream_frames(n_out, ch, 24000, kb) < frames:
            n_out += 1
        assert M.stream_frames(n_out, ch, 24000, kb) == frames
        paths = {"resampled": (48000, 2 * n_out, True), "native": (24000, n_out, False)}
        bufs = {}
        for p, (sr, n, rs) in paths.items():
            l, r = make_signal("noise", n, sr, seed=5)
            pcm = np.concatenate([l, r])                # every stream of the batch reads this one signal
            nb = M.stream_bytes(ch, sr, kb, n, resample=rs)
            assert nb > 0
            bufs[p] = dict(sr=sr, n=n, rs=rs, nb=nb, d_pcm=torch.from_numpy(pcm).cuda(), d_out=torch.empty(S * nb, dtype=torch.uint8, device="cuda"),
                           pcm_off=[0] * S, ns=[n] * S, out_off=[nb * s for s in range(S)], step=[], rs_ms=[])
        for it in range(args.warmup + args.steps):
            for p, b in bufs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tm = M.encode_streams_device(ch, b["sr"], kb, b["d_pcm"].data_ptr(), b["pcm_off"], b["ns"], b["d_out"].data_ptr(),
                                             b["out_off"], resample=b["rs"])
                dt = (time.perf_counter() - t0) * 1e3
                if it >= args.warmup:
                    b["step"].append(dt)
                    b["rs_ms"].append(float(tm[14]))
        out = {}
        for p, b in bufs.items():
            step = statistics.median(b["step"])
            audio_s = S * b["n"] / b["sr"]
            out[p] = {"step_ms": round(step, 3), "resampler_ms": round(statistics.median(b["rs_ms"]), 4),
                      "audio_s_per_s": round(audio_s / (step / 1e3), 1), "streams": S, "input_samples_per_stream": b["n"]}
        out["frames_per_stream"] = frames
        out["same_output_bytes_per_stream"] = bufs["resampled"]["nb"] == bufs["native"]["nb"]
        out["resampling_overhead_pct"] = round(100.0 * (out["resampled"]["step_ms"] / out["native"]["step_ms"] - 1.0), 2)
        res[name] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
