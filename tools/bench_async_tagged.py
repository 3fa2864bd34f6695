#!/usr/bin/env python3
"""Finished files from an encode session (mp3b200_encode_streams_tagged_async, DESIGN.md 15) against the synchronous tagged
device call (mp3b200_encode_streams_tagged_device) on the same device buffers, each with and without ReplayGain.

Two workloads:
  c2    one stereo 44.1 kHz 128 kbps sweep of 10 001 frames (Int16)
  c3    100 stereo 48 kHz 320 kbps streams of 1000 white-noise frames (Int16; 16 distinct streams, cycled)
Every shape is warmed first.  Then, for each workload and each of {tag, tag + ReplayGain}, in one run with the arms
alternating:
  wall      N back-to-back calls then one synchronise: the session (N output buffers) against N synchronous calls; median
            and minimum ms per call over the rounds
  enqueue   host time of one session call while the session's stream is held busy by a spin kernel, so that nothing but
            the enqueue is timed
The output buffers, lengths and gains of both arms are compared.  Prints the device name and power limit, read in the same
run, with the numbers, and one JSON line at the end.

  python tools/bench_async_tagged.py --calls 10 --rounds 7
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bench_async import power_limit_w  # noqa: E402


class Work:
    def __init__(self, M, torch, ch, sr, kbps, rows):
        self.cfg = (ch, sr, kbps)
        self.ns = np.array([len(l) for l, _ in rows], dtype=np.int64)
        host = np.concatenate([np.concatenate([l, r]) for l, r in rows] + [np.zeros(8, np.int16)])
        self.pcm = torch.from_numpy(host).cuda()
        self.pcm_off = np.cumsum([0] + [n * ch for n in self.ns])[:-1].astype(np.int64)
        tfs = M.lametag_size(ch, sr, kbps)
        room = np.array([M.stream_bytes(ch, sr, kbps, int(n)) + tfs for n in self.ns], dtype=np.int64)
        self.out_off = np.cumsum([0] + list(room))[:-1].astype(np.int64)
        self.out_len = int(room.sum()) + 8

    def sync_call(self, M, out, rg):
        return M.encode_streams_device_tagged(*self.cfg, self.pcm.data_ptr(), self.pcm_off, self.ns, out.data_ptr(), self.out_off,
                                              find_replay_gain=rg)

    def async_call(self, sess, out, rg):
        return sess.encode_streams_tagged(*self.cfg, self.pcm, self.pcm_off, self.ns, out, self.out_off, find_replay_gain=rg)


def measure(M, torch, name, w, rg, calls, rounds, sess):
    s = sess.stream
    outs = [torch.zeros(w.out_len, dtype=torch.uint8, device="cuda") for _ in range(calls)]
    ref = torch.zeros(w.out_len, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ref_ob, title, album = w.sync_call(M, ref, rg)
    ob, gains, st = w.async_call(sess, outs[0], rg)     # warm: workspace, staging, both loop graphs
    M.check_status(st)
    same = ob == ref_ob and (not rg or gains.cpu().tolist() == title + [album])
    rg_passes = int(st.cpu()[4])
    enq = []
    for _ in range(rounds * 3):
        with torch.cuda.stream(s):
            torch.cuda._sleep(50_000_000)
        t0 = time.perf_counter()
        _, _, st = w.async_call(sess, outs[0], rg)
        enq.append((time.perf_counter() - t0) * 1e3)
        s.synchronize()
        M.check_status(st)
    wall = {"async": [], "sync": []}
    for r in range(rounds):
        for arm in (("async", "sync") if r % 2 == 0 else ("sync", "async")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if arm == "async":
                sts = [w.async_call(sess, o, rg)[2] for o in outs]
                s.synchronize()
            else:
                for o in outs:
                    w.sync_call(M, o, rg)
            wall[arm].append((time.perf_counter() - t0) * 1e3 / calls)
            if arm == "async":
                for st in sts:
                    M.check_status(st)
            same = same and all(torch.equal(o, ref) for o in outs)
    res = {"enqueue_ms_median": statistics.median(enq), "enqueue_ms_max": max(enq),
           "wall_ms_per_call_median": {k: statistics.median(v) for k, v in wall.items()},
           "wall_ms_per_call_min": {k: min(v) for k, v in wall.items()}, "replaygain_passes": rg_passes,
           "calls": calls, "rounds": rounds, "results_equal": same}
    print(name, json.dumps(res), flush=True)
    assert same, "the session's files, lengths or gains differ from the synchronous call's"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10, help="back-to-back calls per timed window")
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    import torch

    import lamejs_b200 as M
    from synth import sweep, white

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}
    print("device", res, flush=True)
    sess = M.EncodeSession(torch.cuda.Stream())
    c2 = Work(M, torch, 2, 44100, 128, [sweep(10000 * 1152, 44100)])
    distinct = [white(999 * 1152, 300 + i) for i in range(16)]
    c3 = Work(M, torch, 2, 48000, 320, [distinct[i % 16] for i in range(100)])
    for name, w in (("c2", c2), ("c3", c3)):
        for rg in (False, True):
            key = name + ("_replaygain" if rg else "_tag")
            res[key] = measure(M, torch, key, w, rg, a.calls, a.rounds, sess)
    sess.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
