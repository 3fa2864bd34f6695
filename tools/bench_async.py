#!/usr/bin/env python3
"""Cost and gain of encode sessions (mp3b200_encode_streams_async, DESIGN.md 14) against the synchronous device batch
(mp3b200_encode_streams_device_ex) on the same device buffers.

Two workloads:
  c2    one stereo 44.1 kHz 128 kbps sweep of 10 001 frames (Int16)
  live  512 mono streams at 24 kHz 64 kbps (a native configuration), 100 ms each (2400 samples)
For each, in one run, the arms alternate:
  enqueue   host time of one async call of a warm shape while the session's stream is held busy by a spin kernel, so that
            nothing but the enqueue is timed
  wall      N back-to-back calls then one synchronise: async (one session, N output buffers) against N synchronous calls;
            median ms per call over the rounds
and, once per workload, the one-off host cost of the first call of a new shape in a warm session (the fixed-point loop
graph is captured and instantiated), against the same call once the shape is warm.  Bytes of both arms are compared.
Prints the device name and power limit with the numbers and one JSON line at the end.

  python tools/bench_async.py --calls 20 --rounds 7
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


class Work:
    def __init__(self, M, torch, ch, sr, kbps, rows):
        self.cfg = (ch, sr, kbps)
        self.ns = np.array([len(l) for l, _ in rows], dtype=np.int64)
        host = np.concatenate([np.concatenate([l, r]) if ch == 2 else l for l, r in rows] + [np.zeros(8, np.int16)])
        self.pcm = torch.from_numpy(host).cuda()
        self.pcm_off = np.cumsum([0] + [n * ch for n in self.ns])[:-1].astype(np.int64)
        nbs = {int(n): M.stream_bytes(ch, sr, kbps, int(n)) for n in np.unique(self.ns)}
        nb = np.array([nbs[int(n)] for n in self.ns], dtype=np.int64)
        self.out_off = np.cumsum([0] + list(nb))[:-1].astype(np.int64)
        self.out_len = int(nb.sum()) + 8

    def sync_call(self, M, out):
        M.encode_streams_device(*self.cfg, self.pcm.data_ptr(), self.pcm_off, self.ns, out.data_ptr(), self.out_off)

    def async_call(self, sess, out, ns=None):
        return sess.encode_streams(*self.cfg, self.pcm, self.pcm_off, self.ns if ns is None else ns, out, self.out_off)


def measure(M, torch, name, w, calls, rounds, sess):
    s = sess.stream
    outs = [torch.zeros(w.out_len, dtype=torch.uint8, device="cuda") for _ in range(calls)]
    ref = torch.zeros(w.out_len, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    w.sync_call(M, ref)
    M.check_status(w.async_call(sess, outs[0]))     # warm: workspace, staging, loop graph
    torch.cuda.synchronize()
    # enqueue: the stream is busy with a spin kernel while the call is timed
    enq = []
    for _ in range(rounds * 3):
        with torch.cuda.stream(s):
            torch.cuda._sleep(50_000_000)
        t0 = time.perf_counter()
        st = w.async_call(sess, outs[0])
        enq.append((time.perf_counter() - t0) * 1e3)
        s.synchronize()
        M.check_status(st)
    # wall time of `calls` back-to-back calls, the arms alternating
    wall = {"async": [], "sync": []}
    for r in range(rounds):
        for arm in (("async", "sync") if r % 2 == 0 else ("sync", "async")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if arm == "async":
                sts = [w.async_call(sess, o) for o in outs]
                s.synchronize()
            else:
                for o in outs:
                    w.sync_call(M, o)
            wall[arm].append((time.perf_counter() - t0) * 1e3 / calls)
            if arm == "async":
                for st in sts:
                    M.check_status(st)
    same = all(torch.equal(o, ref) for o in outs)
    res = {"enqueue_ms_median": statistics.median(enq), "enqueue_ms_max": max(enq),
           "wall_ms_per_call_median": {k: statistics.median(v) for k, v in wall.items()},
           "wall_ms_per_call_min": {k: min(v) for k, v in wall.items()}, "calls": calls, "rounds": rounds, "bytes_equal": same}
    print(name, json.dumps(res), flush=True)
    return res


def capture_cost(M, torch, w, sess, shrink):
    """host ms of the first call of a new shape (shorter streams: no workspace growth) and of the same call warm"""
    ns = np.maximum(w.ns - shrink, 0)
    out = torch.zeros(w.out_len, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    t = []
    for _ in range(2):
        t0 = time.perf_counter()
        st = w.async_call(sess, out, ns)
        t.append((time.perf_counter() - t0) * 1e3)
        torch.cuda.synchronize()
        M.check_status(st)
    return {"first_call_ms": t[0], "warm_call_ms": t[1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20, help="back-to-back calls per timed window")
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    import torch

    import lamejs_b200 as M
    from synth import make_signal, sweep

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}
    print("device", res, flush=True)
    sess = M.EncodeSession(torch.cuda.Stream())

    l, r = sweep(10000 * 1152, 44100)
    c2 = Work(M, torch, 2, 44100, 128, [(l, r)])
    res["c2"] = measure(M, torch, "c2", c2, a.calls, a.rounds, sess)
    res["c2"]["new_shape"] = capture_cost(M, torch, c2, sess, 1152 * 500)

    kb = 64 if M.out_samplerate(1, 24000, 64) == 24000 else 48
    live = Work(M, torch, 1, 24000, kb, [(make_signal("noise", 2400, 24000, 100 + i)[0], None) for i in range(512)])
    res["live"] = measure(M, torch, "live", live, a.calls, a.rounds, sess)
    res["live"]["kbps"] = kb
    res["live"]["new_shape"] = capture_cost(M, torch, live, sess, 600)
    sess.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
