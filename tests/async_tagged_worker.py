"""Runs in a subprocess of tests/test_gpu_async_tagged.py with MP3B200_LIB naming a library whose ReplayGain speculation is
built to need many repair passes (lamejs_b200.lib() is a process singleton, so one process per library).  Encodes one
C2-length stream through a session's tagged call with the analysis, twice (the second call reuses the captured graph), and
prints one JSON line: {"sha256": of the output buffer, "gains": [...], "status": the 8 words, "sync_passes": the pass
count of the synchronous analysis}."""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from synth import make_signal  # noqa: E402
from test_gpu_async_tagged import Tagged  # noqa: E402


def main():
    import torch

    import lamejs_b200 as M

    assert os.path.samefile(M.lib()._name, os.environ["MP3B200_LIB"])
    l, r = make_signal("sweep", 10000 * 1152, 44100, seed=1)
    b = Tagged(M, 2, 44100, 128, [(l, r)])
    sync_passes = b.rg_passes(M)
    res = []
    with M.EncodeSession(torch.cuda.Stream()) as sess:
        sess.stream.wait_stream(torch.cuda.current_stream())
        for _ in range(2):
            with torch.cuda.stream(sess.stream):
                o = b.out()
            _, gains, st = b.run(sess, o, True)
            M.check_status(st)
            res.append((hashlib.sha256(o.cpu().numpy().tobytes()).hexdigest(), gains.cpu().tolist(), st.cpu().tolist()))
    assert res[0] == res[1], res
    print(json.dumps({"sha256": res[0][0], "gains": res[0][1], "status": res[0][2], "sync_passes": sync_passes}))


if __name__ == "__main__":
    main()
