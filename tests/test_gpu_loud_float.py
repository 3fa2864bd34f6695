"""Loud Float32 input on the GPU against lamejs itself (tests/golden/lamejs_loud_golden.json): a handle with the fixture's
call schedule, host, device and tagged whole streams, and the ReplayGain fixtures through handles and whole streams.  Where
lamejs encodes, the bytes and per-call sizes are lamejs's; where it throws (a frame's bits do not fit its slot), the
library refuses the same call with MP3B200_ERR_CONFIG, k_q_pack has not packed the frame, and a refused handle call leaves
every handle of the call as it was.  Samples beyond 2^35 once scaled (beyond 2^20 x full scale) are refused by the input
gate.  The loudest encodable rung of each configuration is compared with the oracle stage by stage."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import float_signals as FS  # noqa: E402
import oracle_f32  # noqa: E402
import stage_taps  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_loud_golden.json")))
GATE = 2.0 ** 35                       # MP3_F32_MAX_SAMPLE (k_resample.cuh)
FRACTIONAL = (44100, 22050, 11025)     # see tests/test_float_golden_cpu.py


def gated(c):
    return FS.loud_peak(c) > GATE


def cfg_of(c):
    return c["channels"], c["samplerate"], c["kbps"]


ENCODED = sorted(n for n, c in GOLDEN.items() if not c["rg"] and not gated(c))
REPLAYGAIN = sorted(n for n, c in GOLDEN.items() if c["rg"] and not gated(c))
REFUSED_AT_GATE = sorted(n for n, c in GOLDEN.items() if not c["rg"] and gated(c))


def loudest_encodable():
    """per configuration, the loudest rung below the gate that lamejs encodes whole"""
    best = {}
    for n in ENCODED:
        c = GOLDEN[n]
        if c["thrown"] is None and (cfg_of(c) not in best or c["magnitude"] > GOLDEN[best[cfg_of(c)]]["magnitude"]):
            best[cfg_of(c)] = n
    return sorted(best.values())


@pytest.fixture(scope="module")
def M():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import lamejs_b200
    return lamejs_b200


def sha(b):
    return hashlib.sha256(b).hexdigest()


def rows(c):
    l, r, calls = FS.loud_case_signal(c)
    return l.astype(np.float32), None if r is None else r.astype(np.float32), calls


def test_golden_splits_at_the_gate():
    assert len(ENCODED) > 100 and len(REFUSED_AT_GATE) > 50 and len(REPLAYGAIN) >= 6
    assert any(GOLDEN[n]["thrown"] is not None for n in ENCODED) and any(GOLDEN[n]["thrown"] is None for n in ENCODED)
    # the loudest rung below the gate holds streams lamejs encodes
    assert any(GOLDEN[n]["thrown"] is None and GOLDEN[n]["magnitude"] == 2 ** 20 for n in ENCODED)
    assert len(loudest_encodable()) == len({cfg_of(GOLDEN[n]) for n in ENCODED})


@pytest.mark.parametrize("name", ENCODED)
def test_fixture_encodes_or_is_refused_like_lamejs(M, name):
    import torch

    c = GOLDEN[name]
    ch, sr, kb = cfg_of(c)
    rs = M.out_samplerate(ch, sr, kb) != sr
    lf, rf, calls = rows(c)
    # the handle with the fixture's calls: lamejs's sizes up to the call that threw, which is refused
    e = M.Mp3Encoder(ch, sr, kb, resample=rs)
    out = []
    for i, x in enumerate(calls):
        if i == c["thrown"]:
            before = e.export_state()
            with pytest.raises(M.Mp3B200Error, match="bit budget"):
                e.flush() if x is None else e.encodeBuffer(*x)
            assert e.export_state() == before, name
            break
        out.append(e.flush() if x is None else e.encodeBuffer(*x))
    e.close()
    assert [len(b) for b in out] == c["sizes"] and sha(b"".join(out)) == c["sha256"], name
    # whole streams, host, device and tagged: lamejs's stream, or a refusal when any of its frames is over budget
    rr = None if rf is None else [rf]
    pcm = np.concatenate([lf, rf]) if ch == 2 else lf
    nb = M.stream_bytes(ch, sr, kb, len(lf), resample=rs)
    d_pcm = torch.from_numpy(pcm).cuda()
    d_out = torch.zeros(nb, dtype=torch.uint8, device="cuda")
    if c["thrown"] is None:
        assert sha(M.encode_streams(ch, sr, kb, [lf], rr, resample=rs)[0]) == c["sha256"], name
        M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [len(lf)], d_out.data_ptr(), [0], resample=rs, float32=True)
        assert sha(d_out.cpu().numpy().tobytes()) == c["sha256"], name
        tagged = M.encode_streams_tagged(ch, sr, kb, [lf], rr, resample=rs)[0]
        assert sha(tagged[len(tagged) - c["bytes"]:]) == c["sha256"], name
    else:
        with pytest.raises(M.Mp3B200Error, match="bit budget"):
            M.encode_streams(ch, sr, kb, [lf], rr, resample=rs)
        with pytest.raises(M.Mp3B200Error, match="bit budget"):
            M.encode_streams_device(ch, sr, kb, d_pcm.data_ptr(), [0], [len(lf)], d_out.data_ptr(), [0], resample=rs,
                                    float32=True)
        with pytest.raises(M.Mp3B200Error, match="bit budget"):
            M.encode_streams_tagged(ch, sr, kb, [lf], rr, resample=rs)
        if c["schedule"][0][0] == c["samples"]:          # one whole call: the stage taps refuse the same stream
            with pytest.raises(M.Mp3B200Error, match="bit budget"):
                M.debug_stages(ch, sr, kb, lf, rf, want=stage_taps.ALL_TAPS, resample=rs)


@pytest.mark.parametrize("name", REPLAYGAIN)
def test_replaygain_fixture(M, name):
    """ReplayGain on: the handle with the fixture's calls (refused at lamejs's call, or lamejs's bytes, RadioGain and tag
    field), and the tagged whole stream with its analysis"""
    c = GOLDEN[name]
    ch, sr, kb = cfg_of(c)
    assert M.out_samplerate(ch, sr, kb) == sr and sr not in FRACTIONAL
    lf, rf, calls = rows(c)
    e = M.Mp3Encoder(ch, sr, kb, write_vbr_tag=True, find_replay_gain=True)
    out = []
    for i, x in enumerate(calls):
        if i == c["thrown"]:                       # (state blobs do not carry the ReplayGain analysis: see the batch test)
            with pytest.raises(M.Mp3B200Error, match="bit budget"):
                e.flush() if x is None else e.encodeBuffer(*x)
            break
        out.append(e.flush() if x is None else e.encodeBuffer(*x))
    assert [len(b) for b in out] == c["sizes"] and sha(b"".join(out)) == c["sha256"], name
    if c["thrown"] is not None:
        e.close()
        with pytest.raises(M.Mp3B200Error, match="bit budget"):
            M.encode_streams_replaygain(ch, sr, kb, [lf], None if rf is None else [rf])
        return
    at = 4 + ((32 if ch == 2 else 17) if sr >= 32000 else (17 if ch == 2 else 9)) + 116 + 19
    field = bytes.fromhex(c["tag"])[at:at + 2]
    tag = e.lametag_frame()
    assert e.replay_gain[1] == c["radio_gain"][-1] and tag[at:at + 2] == field, name
    e.close()
    streams, title, _ = M.encode_streams_replaygain(ch, sr, kb, [lf], None if rf is None else [rf])
    assert M.radio_gain(title[0]) == c["radio_gain"][-1] and streams[0][:len(tag)] == tag, name
    assert sha(streams[0][len(tag):]) == sha(b"".join(out)[len(tag):]), name


@pytest.mark.parametrize("rg", [False, True], ids=["plain", "replaygain"])
def test_refused_batch_call_leaves_every_handle_as_it_was(M, rg):
    """A loud handle batched with a quiet one: the call that reaches an over-budget frame is refused as a whole, both
    handles export the state they had before it, and quiet input then continues as if the loud call had never been made --
    the bytes (and with ReplayGain the title gain and tag) of the oracle / a handle that never saw it."""
    ch, sr, kb = 2, 32000, 128
    q = lambda n, seed: FS.loud("burst", 1, n, sr, seed, 1.0)                   # noqa: E731  full scale
    # the input of fixture rg_burst_262144_2_32000_128_whole, on which lamejs throws in its first call
    loud_l, loud_r = FS.loud("burst", 2 ** 18, sr // 4 + 101, sr, 2000, 0.95)
    a1, a2, b1, b2 = q(3001, 1), q(2500, 2), q(2002, 3), q(1900, 4)
    f32 = lambda x: x.astype(np.float32)                                        # noqa: E731
    kw = dict(write_vbr_tag=rg, find_replay_gain=rg)
    A, B = M.Mp3Encoder(ch, sr, kb, **kw), M.Mp3Encoder(ch, sr, kb, **kw)
    outA, outB = [], []
    for o, x in zip((outA, outB), M.encode_batch([A, B], [f32(a1[0]), f32(b1[0])], [f32(a1[1]), f32(b1[1])])):
        o.append(x)
    state = lambda: None if rg else (A.export_state(), B.export_state())        # noqa: E731  (blobs carry no ReplayGain)
    before = state()
    with pytest.raises(M.Mp3B200Error, match="bit budget"):
        M.encode_batch([A, B], [f32(loud_l), f32(b2[0])], [f32(loud_r), f32(b2[1])])
    assert state() == before
    for o, x in zip((outA, outB), M.encode_batch([A, B], [f32(a2[0]), f32(b2[0])], [f32(a2[1]), f32(b2[1])])):
        o.append(x)
    for o, x in zip((outA, outB), M.flush_batch([A, B])):
        o.append(x)
    # references that never saw the loud call
    for out, (x1, x2), h in ((outA, (a1, a2), A), (outB, (b1, b2), B)):
        calls = [(f32(x1[0]), f32(x1[1])), (f32(x2[0]), f32(x2[1]))]
        ref, sizes, _, _ = oracle_f32.encode_calls(ch, sr, kb, calls, write_vbr_tag=rg)
        assert [len(b) for b in out] == sizes and b"".join(out) == ref
        if rg:
            R = M.Mp3Encoder(ch, sr, kb, **kw)
            for x in calls:
                R.encodeBuffer(*x)
            R.flush()
            assert h.replay_gain == R.replay_gain and h.lametag_frame() == R.lametag_frame()
            R.close()
    A.close()
    B.close()


@pytest.mark.parametrize("name", loudest_encodable())
def test_loudest_encodable_rung_matches_the_oracle_stage_by_stage(M, name):
    """xr, block types, masking, ATH adjust, l3_enc, side info and the quantizer state bit-equal to the oracle's traces where
    the rate loop works at the top of the gain range"""
    c = GOLDEN[name]
    ch, sr, kb = cfg_of(c)
    rs = M.out_samplerate(ch, sr, kb) != sr
    lf, rf, _ = rows(c)
    G = M.granules_per_frame(ch, sr, kb, resample=rs)
    F = M.stream_frames(len(lf), ch, sr, kb, resample=rs)
    ref, _, tr = oracle_f32.encode_stream(ch, sr, kb, lf, rf, trace_frames=F + 2)
    assert len(tr) == F and sha(ref) == c["sha256"]
    g = M.debug_stages(ch, sr, kb, lf, rf, want=stage_taps.ALL_TAPS, resample=rs)
    stage_taps.compare(g, tr, ref, G, ch, name)


@pytest.mark.parametrize("name", REFUSED_AT_GATE)
def test_input_beyond_the_gate_is_refused(M, name):
    c = GOLDEN[name]
    ch, sr, kb = cfg_of(c)
    rs = M.out_samplerate(ch, sr, kb) != sr
    lf, rf, _ = rows(c)
    with pytest.raises(M.Mp3B200Error, match="2\\^35"):
        M.encode_streams(ch, sr, kb, [lf], None if rf is None else [rf], resample=rs)
    e = M.Mp3Encoder(ch, sr, kb, resample=rs)
    before = e.export_state()
    with pytest.raises(M.Mp3B200Error, match="2\\^35"):
        e.encodeBuffer(lf, rf)
    assert e.export_state() == before
    e.close()


def test_seek_refuses_history_beyond_the_gate(M):
    """seek only sets a handle's state (it encodes nothing): its history is refused at the gate, and the handle stays fresh"""
    ch, sr, kb = 2, 44100, 128
    frame, fs = 5, 1152
    n = frame * fs + 224 - (frame * fs - 1104)
    l, r = FS.loud("noise", 1e9, n, sr, 3, 1.0)
    e = M.Mp3Encoder(ch, sr, kb)
    before = e.export_state()
    with pytest.raises(M.Mp3B200Error, match="2\\^35"):
        e.seek(frame, l.astype(np.float32), r.astype(np.float32))
    assert e.export_state() == before
    e.seek(frame, (l / 1e9).astype(np.float32), (r / 1e9).astype(np.float32))
    e.close()
