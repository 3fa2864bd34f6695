"""ReplayGain (lamejs findReplayGain) on the CPU: the restatement in tests/replaygain_ref.cpp against lamejs itself
(tests/golden/lamejs_replaygain_golden.json), against a float64 filter, and the dependence of the sums on the pieces."""
import hashlib
import json
import os

import numpy as np
import pytest
from scipy import signal as sps

import oracle_lib
import replaygain_ref as RG
from synth import make_signal

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "lamejs_replaygain_golden.json")))


def _schedule(c):
    return [("flush",) if s < 0 else ("enc", s) for s in c["schedule"]]


def _sideinfo_len(ch, out_sr):
    """header + side info in front of the tag's "Info" (MPEG-1: 32 / 17 bytes of side info, MPEG-2 / 2.5: 17 / 9)"""
    return 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9))


@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_matches_lamejs(name):
    c = GOLDEN[name]
    l, r = make_signal(c["kind"], c["samples"], c["samplerate"], seed=c["seed"])
    res = RG.analyze_stream(c["channels"], c["samplerate"], c["kbps"], l, r if c["channels"] == 2 else None, schedule=_schedule(c))
    sums = np.concatenate([w[:, :2] for w in res.windows]) if res.windows else np.zeros((0, 2), np.uint64)
    assert len(sums) == c["windows"]
    assert hashlib.sha256(np.ascontiguousarray(sums, dtype="<u8").tobytes()).hexdigest() == c["windows_sha256"]
    assert res.radio == c["radio_gain"]
    out_sr = oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"])
    tag = bytes.fromhex(c["tag"])
    at = _sideinfo_len(c["channels"], out_sr) + 116 + 19
    assert int.from_bytes(tag[at:at + 2], "big") == RG.tag_field(res.radio[-1])
    assert tag[at - 4:at] == b"\0\0\0\0"          # the peak amplitude stays 0 (it needs the decoder)
    calls = [s for s in c["schedule"] if s >= 0]
    # the audio does not depend on the analysis (at 44.1 / 22.05 / 11.025 kHz lamejs's own tagged stream differs from the
    # oracle's anyway: its frame size is a fraction there, tests/test_tag_oracle.py)
    if c["schedule"].count(-1) == 1 and len(set(calls[:-1])) <= 1 and out_sr not in (44100, 22050, 11025):
        data, _, _ = oracle_lib.encode_stream_tagged(c["channels"], c["samplerate"], c["kbps"], l, r if c["channels"] == 2 else None,
                                                     chunk=calls[0] if len(calls) > 1 else None)
        assert hashlib.sha256(data).hexdigest() == c["sha256"]


def test_golden_covers_the_issue():
    rates = {oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"]) for c in GOLDEN.values()}
    assert rates == set(RG.RATES)
    assert any(oracle_lib.out_samplerate(c["channels"], c["samplerate"], c["kbps"]) != c["samplerate"] for c in GOLDEN.values())
    assert {c["channels"] for c in GOLDEN.values()} == {1, 2}
    assert any(c["radio_gain"] == [RG.radio_gain(RG.GAIN_NOT_ENOUGH_SAMPLES)] for c in GOLDEN.values())
    assert any(len(c["radio_gain"]) == 2 for c in GOLDEN.values())
    assert any(c["fdlibm"] for c in GOLDEN.values())
    assert any(0 < s < 10 for c in GOLDEN.values() for s in c["schedule"])


def test_not_enough_samples_clamps():
    assert RG.radio_gain(RG.GAIN_NOT_ENOUGH_SAMPLES) == -246010
    assert RG.tag_field(-246010) == 0x2000 | 0xC00 | 0x200 | 0x1FE


@pytest.mark.parametrize("ch,sr,kbps", [(2, 44100, 128), (1, 22050, 64), (2, 8000, 24), (2, 48000, 64)])
def test_windows_agree_with_float64_filters(ch, sr, kbps):
    """the Float32-rounded cascade stays within a tight tolerance of the same filters in float64"""
    l, r = make_signal("noise", sr, sr, seed=7)
    rows, out_sr, titles = RG.analysed(ch, sr, kbps, l, r if ch == 2 else None, RG.schedule_of(len(l)))
    res = RG.run(rows, out_sr, titles)
    req = RG.RATES.index(out_sr)
    src = open(os.path.join(HERE, "replaygain_ref.cpp")).read()
    yule = np.array(eval("[" + src.split("ABYule[9][21] = {")[1].split("};")[0].replace("{", "[").replace("}", "]") + "]"))[req]
    butter = np.array(eval("[" + src.split("ABButter[9][5] = {")[1].split("};")[0].replace("{", "[").replace("}", "]") + "]"))[req]
    W = RG.sample_window(out_sr)
    k = len(res.windows[0])
    for c in range(ch):
        y = sps.lfilter(yule[0::2], np.concatenate([[1.0], yule[1::2]]), rows[c].astype(np.float64))
        z = sps.lfilter(butter[0::2], np.concatenate([[1.0], butter[1::2]]), y)
        e = (z[:k * W] ** 2).reshape(k, W).sum(axis=1)
        got = res.windows[0][:, c].view(np.float64)
        np.testing.assert_allclose(got, e, rtol=1e-4, atol=1e-3 * W)


def test_pieces_change_the_sum_bits():
    """the same samples analysed in other pieces: the filters agree, the sums' bits do not"""
    l, r = make_signal("white", 3 * 44100, 44100, seed=11)
    a = RG.analyze_stream(2, 44100, 128, l, r)
    odd = [(7, 333, 1000)[i % 3] for i in range(400)]
    odd = odd[:next(i for i in range(len(odd)) if sum(odd[:i + 1]) >= len(l))]
    odd.append(len(l) - sum(odd))
    b = RG.analyze_stream(2, 44100, 128, l, r, chunk=odd)
    assert len(a.windows[0]) == len(b.windows[0])
    assert (a.windows[0][:, :2] != b.windows[0][:, :2]).any()
    same = a.windows[0][:, :2].view(np.float64)
    other = b.windows[0][:, :2].view(np.float64)
    np.testing.assert_allclose(same, other, rtol=1e-12)
