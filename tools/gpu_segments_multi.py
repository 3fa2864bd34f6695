#!/usr/bin/env python3
"""One long stream over N GPUs (torchrun): frames cut into N contiguous ranges, warm-up + verified state hand-over
(lamejs_b200/sharding.py encode_stream_segments).  Checks the gathered bytes against the single-encoder stream and times
both through the same host-buffer handle API (wall clock between barriers, max over ranks).
--tagged: the finished file instead (encode_stream_segments_tagged against encode_streams_replaygain of the whole stream);
--replaygain: with the ReplayGain analysis, which rank 0 runs beside its own range.
  torchrun --nproc-per-node N tools/gpu_segments_multi.py [frames] [warmup] [--tagged] [--replaygain]"""
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import lamejs_b200 as M  # noqa: E402
from lamejs_b200 import sharding  # noqa: E402
from synth import make_signal  # noqa: E402

rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
assert M.lib().mp3b200_set_device(local) == 0
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
flags = [a for a in sys.argv[1:] if a.startswith("--")]
args = [a for a in sys.argv[1:] if not a.startswith("--")]
frames = int(args[0]) if len(args) > 0 else 10000
warmup = int(args[1]) if len(args) > 1 else 8
replaygain = "--replaygain" in flags
tagged = "--tagged" in flags or replaygain
res = {}
for kind in ("sweep", "noise"):
    l, r = make_signal(kind, frames * 1152, 44100)
    mk = lambda: M.Mp3Encoder(2, 44100, 128)

    def single():
        if tagged:
            return M.encode_streams_replaygain(2, 44100, 128, [l], [r], find_replay_gain=replaygain)[0][0]
        e = mk()
        b = e.encodeBuffer(l, r) + e.flush()
        e.close()
        return b

    def segments():
        if tagged:
            return sharding.encode_stream_segments_tagged(2, 44100, 128, l, r, warmup=warmup, find_replay_gain=replaygain,
                                                          device="cuda")[:2]
        return sharding.encode_stream_segments(mk, l, r, 1152, warmup=warmup, device="cuda")

    def barrier():
        dist.barrier()
        torch.cuda.synchronize()

    ref = single()
    t_single = []
    for _ in range(3):
        barrier(); t0 = time.perf_counter(); single(); torch.cuda.synchronize(); t_single.append(time.perf_counter() - t0)
    t_seg, redone = [], 0
    for _ in range(4):
        barrier(); t0 = time.perf_counter()
        got, redone = segments()
        torch.cuda.synchronize()
        dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device="cuda")
        dist.all_reduce(dt, op=dist.ReduceOp.MAX)
        t_seg.append(float(dt.item()))
    if rank == 0:
        res[kind] = {"equal_single_encoder": got == ref, "sha256": hashlib.sha256(got).hexdigest()[:16], "ranges_reencoded": redone,
                     "single_encoder_ms": 1e3 * min(t_single), "segments_ms": 1e3 * min(t_seg[1:]), "speedup": min(t_single) / min(t_seg[1:])}
if rank == 0:
    print(json.dumps({"n_gpus": world, "frames": frames, "warmup_frames": warmup, "tagged": tagged, "replaygain": replaygain,
                      "streams": res}))
dist.destroy_process_group()
