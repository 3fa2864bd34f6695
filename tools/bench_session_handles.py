#!/usr/bin/env python3
"""Live streaming handles in an encode session (DESIGN.md 16) against the synchronous device batch call.

The live workload of tools/bench_device_handles.py: 512 mono handles at a native 24 kHz configuration, fed 100 ms Float32
chunks (2400 samples) that torch makes on the GPU.  Two arms, run alternately in blocks of --rounds rounds on twin handles:
  sync     M.encode_batch(handles, rows of CUDA tensors): each round returns the bytes on the host
  session  EncodeSession.encode_batch(handles, rows): the rounds are queued on the session's stream, which also makes the
           chunks, with no synchronise between them; a host clock spans the block and one synchronise at its end
Reports the median ms per round of each arm, the host time one session call takes to enqueue while its stream is held busy
(median and max), whether the two arms' bytes are identical, and the device name and power limit read in the same run.
--profile DIR also writes a torch.profiler summary of one session block into DIR.

  python tools/bench_session_handles.py --blocks 6 --rounds 50
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
from bench_device_handles import live_kbps, power_limit_w  # noqa: E402

SLEEP_CYCLES = 400_000_000           # torch.cuda._sleep: ~0.2 s on an H100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--handles", type=int, default=512)
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--blocks", type=int, default=6, help="blocks of --rounds rounds per arm, alternated")
    ap.add_argument("--profile", default=None, metavar="DIR")
    a = ap.parse_args()
    import torch
    import lamejs_b200 as M

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w()}
    kb, S, n = live_kbps(M), a.handles, 2400
    st = torch.cuda.Stream()
    sess = M.EncodeSession(st)
    encs = {arm: [M.Mp3Encoder(1, 24000, kb) for _ in range(S)] for arm in ("sync", "session")}
    f = torch.linspace(200.0, 3000.0, S, device="cuda", dtype=torch.float64)[:, None]
    k = torch.arange(n, device="cuda", dtype=torch.float64)[None, :]

    def chunk(r):
        t = (r * n + k) / 24000.0
        return (0.4 * torch.sin(2 * np.pi * f * t) + 0.05 * torch.sin(2 * np.pi * 7.0 * f * t)).float()

    pos = {"sync": 0, "session": 0}
    got = {"sync": [], "session": []}

    def block(arm, keep=True):
        """--rounds rounds of one arm; returns ms per round"""
        torch.cuda.synchronize()
        outs = []
        t0 = time.perf_counter()
        if arm == "sync":
            for _ in range(a.rounds):
                outs.append(M.encode_batch(encs[arm], list(chunk(pos[arm]))))
                pos[arm] += 1
        else:
            with torch.cuda.stream(st):
                for _ in range(a.rounds):
                    x = chunk(pos[arm])
                    outs.append(sess.encode_batch(encs[arm], list(x)))
                    pos[arm] += 1
            st.synchronize()
        dt = (time.perf_counter() - t0) * 1e3 / a.rounds
        if keep:
            got[arm] += outs
        return dt

    block("sync", keep=True)                # warm-up: shapes, graphs, binding
    block("session", keep=True)
    ms = {"sync": [], "session": []}
    for b in range(a.blocks):
        for arm in (("sync", "session") if b % 2 == 0 else ("session", "sync")):
            ms[arm].append(block(arm))

    # enqueue host time with the stream held busy (fewer calls than the session's slots, so none waits for one)
    enq = []
    for _ in range(10):
        x = [chunk(pos["session"] + j) for j in range(3)]
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            torch.cuda._sleep(SLEEP_CYCLES)
        for j in range(3):
            t0 = time.perf_counter()
            got["session"].append(sess.encode_batch(encs["session"], list(x[j])))
            enq.append((time.perf_counter() - t0) * 1e3)
        busy = not st.query()
        st.synchronize()
        for j in range(3):
            got["sync"].append(M.encode_batch(encs["sync"], list(x[j])))
        pos["session"] += 3
        pos["sync"] += 3
        assert busy, "the stream drained before the enqueues were timed"

    same = len(got["sync"]) == len(got["session"])
    for w, (o, off, lens, status) in zip(got["sync"], got["session"]):
        M.check_status(status)
        h = o.cpu().numpy()
        same = same and w == [h[p:p + q].tobytes() for p, q in zip(off, lens)]
    res["live"] = {"handles": S, "kbps": kb, "samples_per_round": n, "rounds_per_block": a.rounds, "blocks": a.blocks,
                   "round_ms_median": {arm: statistics.median(v) for arm, v in ms.items()},
                   "enqueue_ms_busy": {"median": statistics.median(enq), "max": max(enq)}, "bytes_equal": bool(same)}
    print("live", json.dumps(res["live"]), flush=True)

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            block("session", keep=False)
        tab = p.key_averages().table(sort_by="cuda_time_total", row_limit=30)
        with open(os.path.join(a.profile, "profile_session_handles.txt"), "w") as fh:
            fh.write(tab)
        tab = p.key_averages().table(sort_by="cpu_time_total", row_limit=20)
        with open(os.path.join(a.profile, "profile_session_handles_cpu.txt"), "w") as fh:
            fh.write(tab)
    sess.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
