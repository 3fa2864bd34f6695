#!/usr/bin/env python3
"""Phase clocks of k_psy_analysis (PSY_PHASESTAT build): one C2 encode, then cycles per phase of the sampled blocks
(every 16th block of channel 0), median and p90 over the blocks.

  python tools/build_variants.py stat=PSY_PHASESTAT
  MP3B200_LIB=lamejs_b200/libmp3b200_stat.so python tools/psy_phasestat.py

Each phase ends at a block barrier, timed by thread 0.  "partition 1 wait" is thread 0 waiting at the barrier after the
first partition phase, "chain tail" the time the last loudness chain runs on after thread 0 has finished: both are the
block waiting for its loudness thread(s)."""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import lamejs_b200 as M  # noqa: E402
from synth import make_signal  # noqa: E402

ROWS, COLS = 4096, 13
frames = 10000
n = frames * 1152
l, r = make_signal("sweep", n, 44100)
pcm = torch.from_numpy(np.concatenate([l, r])).cuda()
nb = M.stream_bytes(2, 44100, 128, n)
out = torch.zeros(nb + 64, dtype=torch.uint8, device="cuda")
L = M.lib()
if not hasattr(L, "mp3b200_debug_psystat"):
    raise SystemExit("not a PSY_PHASESTAT build (set MP3B200_LIB)")
for _ in range(2):
    M.encode_streams_device(2, 44100, 128, pcm.data_ptr(), [0], [n], out.data_ptr(), [0])
torch.cuda.synchronize()
buf = np.zeros((ROWS, COLS), dtype=np.int64)
rows = L.mp3b200_debug_psystat(buf.ctypes.data_as(ctypes.c_void_p), ROWS)
c = buf[(buf[:, 0] != 0) & (buf[:, 10] != 0) & (buf[:, 12] != 0)]
d = lambda a, b: (c[:, b] - c[:, a]).astype(float)  # noqa: E731
phases = [("load span", d(0, 1)), ("HPF + first pass", d(1, 2)), ("FHT stage 0 + peaks", d(2, 3)),
          ("FHT stage 1", d(3, 4)), ("FHT stage 2", d(4, 5)), ("FHT stage 3", d(5, 6)), ("energies", d(6, 7)),
          ("partition 1 (thread 0)", d(7, 8)), ("partition 1 wait", d(8, 9)), ("partition 2 (thread 0)", d(9, 10)),
          ("chain tail", np.maximum(d(10, 12), 0.0))]
total = np.maximum(c[:, 10], c[:, 12]).astype(float) - c[:, 0]
print("lib:", os.environ.get("MP3B200_LIB", "default"), "blocks sampled:", len(c))
print("%-24s %9s %9s %7s" % ("phase", "median", "p90", "share"))
for name, v in phases + [("block total", total)]:
    print("%-24s %9.0f %9.0f %6.1f%%" % (name, np.median(v), np.percentile(v, 90), 100 * np.median(v) / np.median(total)))
wait = d(8, 9) + np.maximum(d(10, 12), 0.0)
print("waiting on the loudness chain: median %.0f cycles, %.1f %% of the block" % (np.median(wait), 100 * np.median(wait / total)))
