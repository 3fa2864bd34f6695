"""Every lamejs Float32 fixture (tests/golden/lamejs_float_golden.json) through every entry point on the GPU: a handle with
the fixture's call schedule, a batch, host and device whole streams, and, for the ReplayGain fixtures, tagged whole streams
with their title gains and the tag's Radio Replay Gain field."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import float_signals as FS  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_float_golden.json")))
FRACTIONAL = (44100, 22050, 11025)     # see tests/test_float_golden_cpu.py


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def sha(b):
    return hashlib.sha256(b).hexdigest()


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_fixture_through_every_entry_point(M, name):
    import torch

    c = GOLDEN[name]
    ch, sr, kb = c["channels"], c["samplerate"], c["kbps"]
    rs = M.out_samplerate(ch, sr, kb) != sr
    l, r, calls = FS.case_signal(c)
    lf = l.astype(np.float32)
    rf = None if r is None else r.astype(np.float32)
    if c["rg"]:
        streams, title, _ = M.encode_streams_replaygain(ch, sr, kb, [lf], None if rf is None else [rf], resample=rs)
        # lamejs's tag frame as the driver records it: its Radio Replay Gain field (the rest of the frame is the tag writer's,
        # pinned by tests/golden/lamejs_tag_golden.json)
        out_sr = M.out_samplerate(ch, sr, kb)
        at = 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9)) + 116 + 19
        field = bytes.fromhex(c["tag"])[at:at + 2]
        assert M.radio_gain(title[0]) == c["radio_gain"][-1], name
        assert streams[0][at:at + 2] == field, name
        e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, resample=rs, find_replay_gain=True)
        out = [e.encodeBuffer(*x) for x in calls[:-1]] + [e.flush()]
        tag = e.lametag_frame()
        assert e.replay_gain[1] == c["radio_gain"][-1] and tag[at:at + 2] == field and tag == streams[0][:len(tag)], name
        e.close()
        if M.out_samplerate(ch, sr, kb) not in FRACTIONAL:
            assert [len(b) for b in out] == c["sizes"] and sha(b"".join(out)) == c["sha256"], name
        return
    # a handle with the fixture's calls, and the same calls through a batch of two handles
    e = M.Mp3Encoder(ch, sr, kb, resample=rs)
    out = [e.encodeBuffer(*x) for x in calls[:-1]] + [e.flush()]
    e.close()
    assert [len(b) for b in out] == c["sizes"] and sha(b"".join(out)) == c["sha256"], name
    encs = [M.Mp3Encoder(ch, sr, kb, resample=rs) for _ in range(2)]
    parts = [[], []]
    for a, b in calls[:-1]:
        for j, o in enumerate(M.encode_batch(encs, [a, a], None if b is None else [b, b])):
            parts[j].append(o)
    for j, o in enumerate(M.flush_batch(encs)):
        parts[j].append(o)
    for x in encs:
        x.close()
    assert sha(b"".join(parts[0])) == c["sha256"] and sha(b"".join(parts[1])) == c["sha256"], name
    # whole streams: host and device
    assert sha(M.encode_streams(ch, sr, kb, [lf], None if rf is None else [rf], resample=rs)[0]) == c["sha256"], name
    pcm = np.concatenate([lf, rf]) if ch == 2 else lf
    nb = M.stream_bytes(ch, sr, kb, len(lf), resample=rs)
    d_pcm = torch.from_numpy(pcm).cuda()
    d_out = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [len(lf)], d_out.data_ptr(), [0], resample=rs, float32=True)
    assert sha(d_out.cpu().numpy().tobytes()) == c["sha256"], name
