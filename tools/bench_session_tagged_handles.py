#!/usr/bin/env python3
"""Tagged ReplayGain streaming handles in an encode session (DESIGN.md 17) against the synchronous device batch call.

The live workload of tools/bench_session_handles.py with the tag and ReplayGain on: 512 mono handles at a native 24 kHz
configuration (write_vbr_tag=True, find_replay_gain=True), fed 100 ms Float32 chunks (2400 samples) that torch makes on the
GPU.  Two arms, run alternately in blocks of --rounds rounds on twin handles:
  sync     M.encode_batch(handles, rows of CUDA tensors): each round returns the bytes on the host, with the music CRC and
           the ReplayGain analysis finished by host read-backs
  session  EncodeSession.encode_batch_tagged(handles, rows): the rounds are queued on the session's stream, which also makes
           the chunks, with no synchronise between them; a host clock spans the block and one synchronise at its end
Reports the median ms per round of each arm, the host time one session call takes to enqueue while its stream is held busy
(median and max), the loop graphs the session instantiated after warm-up, whether the two arms' bytes, tag frames and gains
(title gains after a flush, and the album gain) are identical, and the device name and power limit read in the same run.
With --profile DIR the invocation measures nothing else: after one warm-up block of the session arm it runs one more under
torch.profiler and reports the GPU time per round and the share of it the ReplayGain copy-in (k_rg_stage_in) and commit
(k_rg_commit) take, with the kernel table written into DIR.  Run it as a process of its own, after the timed run.

  python tools/bench_session_tagged_handles.py --blocks 6 --rounds 50
  python tools/bench_session_tagged_handles.py --rounds 50 --profile DIR
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
    encs = {arm: [M.Mp3Encoder(1, 24000, kb, write_vbr_tag=True, find_replay_gain=True) for _ in range(S)]
            for arm in ("sync", "session")}
    assert all(e.replay_gain_on for e in encs["sync"])
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
                    outs.append(sess.encode_batch_tagged(encs[arm], list(x)))
                    pos[arm] += 1
            st.synchronize()
        dt = (time.perf_counter() - t0) * 1e3 / a.rounds
        if keep:
            got[arm] += outs
        return dt

    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(a.profile, exist_ok=True)
        block("session", keep=False)        # warm-up: shapes, graphs, binding
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            block("session", keep=False)
        ka = p.key_averages()

        def dev_us(e):
            return float(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)))

        kernels = [e for e in ka if dev_us(e) > 0 and e.key.startswith(("_Z", "k_", "void "))]
        total = sum(dev_us(e) for e in ka if dev_us(e) > 0 and "Memcpy" not in e.key and "Memset" not in e.key
                    and not e.key.startswith("cuda"))
        rg = sum(dev_us(e) for e in kernels if "k_rg_stage_in" in e.key or "k_rg_commit" in e.key)
        res["profile"] = {"gpu_ms_per_round": total / 1e3 / a.rounds, "rg_copy_in_and_commit_ms_per_round": rg / 1e3 / a.rounds,
                          "rg_copy_share": rg / total if total else None}
        with open(os.path.join(a.profile, "profile_session_tagged_handles.txt"), "w") as fh:
            fh.write(ka.table(sort_by="cuda_time_total", row_limit=40))
        print("profile", json.dumps(res["profile"]), flush=True)
        sess.close()
        print(json.dumps(res))
        return

    block("sync")                           # warm-up: shapes, graphs, binding
    block("session")
    warm = sess.graph_instantiations()
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
            got["session"].append(sess.encode_batch_tagged(encs["session"], list(x[j])))
            enq.append((time.perf_counter() - t0) * 1e3)
        busy = not st.query()
        st.synchronize()
        for j in range(3):
            got["sync"].append(M.encode_batch(encs["sync"], list(x[j])))
        pos["session"] += 3
        pos["sync"] += 3
        assert busy, "the stream drained before the enqueues were timed"
    graphs_after_warmup = sess.graph_instantiations() - warm

    def bytes_of(o, off, lens):
        h = o.cpu().numpy()
        return [h[p:p + q].tobytes() for p, q in zip(off, lens)]

    for g in got["session"]:
        M.check_status(g[3])
    diff = [j for j, (w, g) in enumerate(zip(got["sync"], got["session"])) if w != bytes_of(*g[:3])]
    eq = {"rounds": len(got["sync"]) == len(got["session"]) and not diff}
    # the end of the streams: flush, tag frames and gains of both arms
    flushed = sess.flush_batch_tagged(encs["session"])
    o, off, lens, status = sess.lametag_frames(encs["session"])
    album, status_a = sess.album_gain(encs["session"])
    st.synchronize()                        # the bytes are read on another stream
    eq["flush"] = M.flush_batch(encs["sync"]) == bytes_of(*flushed[:3])
    M.check_status(status)
    M.check_status(status_a)
    frames = bytes_of(o, off, lens)
    eq["album_gain"] = float(album.cpu()[0]) == M.album_gain(encs["sync"])
    sess.release(encs["session"])
    eq["tag_frames"] = frames == [e.lametag_frame() for e in encs["sync"]]
    eq["title_gains"] = [e.replay_gain for e in encs["session"]] == [e.replay_gain for e in encs["sync"]]
    eq["music_crc"] = [e.music_crc() for e in encs["session"]] == [e.music_crc() for e in encs["sync"]]
    eq["bytes_written"] = [e.bytes_written() for e in encs["session"]] == [e.bytes_written() for e in encs["sync"]]
    res["live"] = {"handles": S, "kbps": kb, "samples_per_round": n, "rounds_per_block": a.rounds, "blocks": a.blocks,
                   "round_ms_median": {arm: statistics.median(v) for arm, v in ms.items()},
                   "enqueue_ms_busy": {"median": statistics.median(enq), "max": max(enq)},
                   "graph_instantiations_after_warmup": graphs_after_warmup, "equal": eq, "first_rounds_differing": diff[:5],
                   "bytes_frames_gains_equal": all(eq.values())}
    print("live", json.dumps(res["live"]), flush=True)

    sess.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
