"""Runs in a subprocess of tests/test_gpu_async.py with MP3B200_LIB naming a library built with bad speculation guesses and
no folded repair (lamejs_b200.lib() is a process singleton, so one process per library): every wrong guess is repaired by
the fixed-point loop, which an encode session runs on the device.  Encodes ragged batches through a session, compares
with the oracle and with encode_streams_device's pass count, and prints one JSON line:
{"fail": [what differed, ...], "passes": {workload: quantizer passes}}."""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import oracle_lib as O  # noqa: E402
from synth import make_signal, white  # noqa: E402


def main():
    import torch

    import lamejs_b200 as M

    assert os.path.samefile(M.lib()._name, os.environ["MP3B200_LIB"])
    fail, passes = [], {}
    sess = M.EncodeSession(torch.cuda.Stream())
    for tag, ch, sr, kbps, frame, rs in (("mpeg1", 2, 44100, 128, 1152, False), ("lsf", 2, 22050, 64, 576, False),
                                         ("lsf_mono", 1, 16000, 24, 576, False), ("resampled", 2, 48000, 64, 1152, True)):
        lens = [1, 700, 1377, 5000, frame * 31 + 5, frame * 64, frame * 150 + 3]
        sigs = []
        for i, n in enumerate(lens):
            l, r = white(n, 0x5EED0050 + i) if i % 3 == 0 else make_signal(("burst", "noise", "sweep")[i % 3], n, sr, 50 + i)
            sigs.append((l, r if ch == 2 else l))
        ns = np.array(lens, dtype=np.int64)
        pcm = np.concatenate([np.concatenate([l, r]) if ch == 2 else l for l, r in sigs] + [np.zeros(8, np.int16)])
        pcm_off = np.cumsum([0] + [n * ch for n in lens])[:-1]
        nb = [M.stream_bytes(ch, sr, kbps, n, rs) for n in lens]
        out_off = np.cumsum([0] + nb)[:-1]
        d_pcm = torch.from_numpy(pcm).cuda()
        ref_out = torch.zeros(sum(nb) + 8, dtype=torch.uint8, device="cuda")
        tm = M.encode_streams_device(ch, sr, kbps, d_pcm.data_ptr(), pcm_off, ns, ref_out.data_ptr(), out_off, resample=rs)
        sess.stream.wait_stream(torch.cuda.current_stream())
        for rep in range(2):                             # the second call of the shape reuses the captured graph
            with torch.cuda.stream(sess.stream):
                d_out = torch.zeros(sum(nb) + 8, dtype=torch.uint8, device="cuda")
            st = sess.encode_streams(ch, sr, kbps, d_pcm, pcm_off, ns, d_out, out_off, resample=rs)
            p = M.check_status(st)
            passes["%s#%d" % (tag, rep)] = p
            if p != int(tm[7]):
                fail.append("%s: %d passes on the device, %d on the host" % (tag, p, int(tm[7])))
            out = d_out.cpu().numpy()
            for i, ((l, r), o, b) in enumerate(zip(sigs, out_off, nb)):
                if out[o:o + b].tobytes() != O.encode_stream(ch, sr, kbps, l, r if ch == 2 else None)[0]:
                    fail.append("%s#%d stream %d (%d samples)" % (tag, rep, i, len(l)))
    sess.close()
    print(json.dumps({"fail": fail, "passes": passes}))


if __name__ == "__main__":
    main()
