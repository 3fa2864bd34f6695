#!/usr/bin/env python3
"""Cost of Float32 input on the device path (encode_streams_device vs encode_streams_device(float32=True)).

For C2 (one stereo 44.1 kHz 128 kbps sweep of 10000 frames) and a c3-shaped batch (stereo 48 kHz 320 kbps, 100 white-noise
streams of 1000 frames) the same samples are kept on the device as Int16 and as Float32 (twice the bytes), and the two
calls are timed alternately in one run: CUDA events around each call on the default stream, and the library's per-stage
timing slots.  Float32 input adds k_stage_f32 and runs the <true> instantiations of the psy analysis and the subband
analysis at the MPEG-1 rate; the output bytes of both must be equal (integer-valued samples).  Prints the device name and
power limit with the numbers.  The host path (encode_streams from host arrays, upload included) is timed the same way.

  python tools/bench_float.py --steps 10 --warmup 3
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

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
        ns = [len(l) for l, _ in sig]
        pcm = np.concatenate([np.concatenate([l, r]) for l, r in sig])
        pcm_off = np.concatenate([[0], np.cumsum([2 * n for n in ns])[:-1]])
        nb = [M.stream_bytes(ch, sr, kb, n) for n in ns]
        out_off = np.concatenate([[0], np.cumsum(nb)[:-1]])
        d_i16 = torch.from_numpy(pcm).cuda()
        d_f32 = d_i16.float()
        outs = {"int16": torch.zeros(sum(nb), dtype=torch.uint8, device="cuda"),
                "float32": torch.zeros(sum(nb), dtype=torch.uint8, device="cuda")}
        src = {"int16": d_i16, "float32": d_f32}

        def run(kind):
            return M.encode_streams_device(ch, sr, kb, src[kind].data_ptr(), pcm_off, ns, outs[kind].data_ptr(), out_off,
                                           float32=(kind == "float32"))

        for _ in range(a.warmup):
            run("int16")
            run("float32")
        ms = {"int16": [], "float32": []}
        slots = {"int16": [], "float32": []}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for i in range(a.steps):
            for kind in (("int16", "float32") if i % 2 == 0 else ("float32", "int16")):
                ev0.record()
                tm = run(kind)
                ev1.record()
                ev1.synchronize()
                ms[kind].append(ev0.elapsed_time(ev1))
                slots[kind].append(tm.tolist())
        torch.cuda.synchronize()
        same = bool(torch.equal(outs["int16"], outs["float32"]))
        med = {k: statistics.median(v) for k, v in ms.items()}
        stage = {k: [statistics.median(s[j] for s in slots[k]) for j in range(16)] for k in slots}
        # host path: PCM uploaded from host memory (Int16 in slices that overlap the psy analysis; Float32 staged whole)
        import time
        hl, hr = [l for l, _ in sig], [r for _, r in sig]
        hlf, hrf = [x.astype(np.float32) for x in hl], [x.astype(np.float32) for x in hr]
        host = {"int16": [], "float32": []}
        for i in range(a.warmup + a.steps):
            for kind in (("int16", "float32") if i % 2 == 0 else ("float32", "int16")):
                t0 = time.perf_counter()
                M.encode_streams(ch, sr, kb, *((hl, hr) if kind == "int16" else (hlf, hrf)))
                if i >= a.warmup:
                    host[kind].append((time.perf_counter() - t0) * 1e3)
        res["workloads"].setdefault(name, {})
        host_med = {k: statistics.median(v) for k, v in host.items()}
        print(name, "host", json.dumps(host_med), flush=True)
        res["workloads"][name] = {"host_call_ms_median": host_med,
            "streams": len(ns), "samples_per_channel": ns[0], "pcm_bytes": {"int16": d_i16.numel() * 2, "float32": d_f32.numel() * 4},
            "call_ms_median": med, "call_ms": ms, "bytes_equal": same,
            "psy_ms_median": {k: stage[k][0] for k in stage}, "scan_subband_ms_median": {k: stage[k][1] for k in stage},
            "pipeline_total_ms_median": {k: stage[k][6] for k in stage},
        }
        print(name, json.dumps(med), "psy", json.dumps(res["workloads"][name]["psy_ms_median"]),
              "scan+subband", json.dumps(res["workloads"][name]["scan_subband_ms_median"]), "bytes_equal", same, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
