"""ReplayGain on the GPU (k_replaygain.cuh) against the CPU restatement of lamejs's analysis (tests/replaygain_ref.py, pinned
against lamejs by tests/test_replaygain_cpu.py): every window's lsum / rsum bits, the histogram, the title and album gains
and the complete tagged bytes."""
import numpy as np
import pytest

import edge_signals
import oracle_lib
import replaygain_ref as RG
from synth import make_signal

pytestmark = pytest.mark.gpu

NATIVE = [(2, 48000, 128), (1, 48000, 128), (2, 44100, 128), (1, 44100, 128), (2, 32000, 128), (1, 32000, 64), (2, 24000, 64),
          (1, 24000, 64), (2, 22050, 64), (1, 22050, 64), (2, 16000, 40), (1, 16000, 40), (2, 12000, 32), (1, 12000, 32),
          (2, 11025, 32), (1, 11025, 32), (2, 8000, 24), (1, 8000, 24)]
RESAMPLED = [(2, 48000, 64), (2, 48000, 40), (2, 32000, 24), (2, 16000, 24), (2, 48000, 24), (2, 24000, 24)]


@pytest.fixture(scope="module")
def enc():
    import lamejs_b200
    return lamejs_b200


def _rs(ch, sr, kb):
    return oracle_lib.out_samplerate(ch, sr, kb) != sr


def _check_windows(enc, ch, sr, kb, l, r):
    rs = _rs(ch, sr, kb)
    got = enc.debug_replaygain(ch, sr, kb, l, r if ch == 2 else None, resample=rs)
    ref = RG.analyze_stream(ch, sr, kb, l, r if ch == 2 else None)
    w = ref.windows[0]
    assert len(got["sums"]) == len(w)
    assert np.array_equal(got["sums"].view(np.uint64), w[:, :2])
    assert np.array_equal(got["idx"], w[:, 2].astype(np.int32))
    assert np.array_equal(got["hist"], ref.hist[0])
    assert got["title_db"] == ref.title_db[0]
    return got, ref


@pytest.mark.parametrize("ch,sr,kb", NATIVE + RESAMPLED)
def test_windows_match_reference(enc, ch, sr, kb):
    l, r = make_signal("noise", sr + 3 * 1152 + 17, sr, seed=sr + ch)
    _check_windows(enc, ch, sr, kb, l, r)


def _patched_tag(stream, ch, out_sr, field):
    """a tagged stream with its Radio Replay Gain field set and the tag CRC recomputed"""
    side = 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9))
    q = side + 116
    b = bytearray(stream)
    b[q + 19:q + 21] = field.to_bytes(2, "big")
    b[q + 38:q + 40] = oracle_lib.crc16(bytes(b[:q + 38])).to_bytes(2, "big")
    return bytes(b)


@pytest.mark.parametrize("ch,sr,kb", [(2, 44100, 128), (1, 8000, 24), (2, 22050, 64), (2, 48000, 64), (2, 32000, 24)])
def test_ragged_batch_bytes_and_album(enc, ch, sr, kb):
    rs = _rs(ch, sr, kb)
    out_sr = oracle_lib.out_samplerate(ch, sr, kb)
    lens = [0, 37, 1152, 5 * 1152 + 1, sr // 2, 2 * sr + 999, 7000]
    kinds = ["noise", "silence", "sweep", "white", "noise", "octave", "burst"]
    sig = [make_signal(k, n, sr, seed=i + 5) for i, (k, n) in enumerate(zip(kinds, lens))]
    lefts = [s[0] for s in sig]
    rights = [s[1] for s in sig] if ch == 2 else None
    plain = enc.encode_streams_tagged(ch, sr, kb, lefts, rights, resample=rs)
    streams, title, album = enc.encode_streams_replaygain(ch, sr, kb, lefts, rights, resample=rs)
    hist = np.zeros(RG.HIST, dtype=np.int64)
    for i in range(len(lens)):
        ref = RG.analyze_stream(ch, sr, kb, lefts[i], rights[i] if ch == 2 else None)
        assert title[i] == ref.title_db[0], i
        hist += ref.hist[0]
        assert streams[i] == _patched_tag(plain[i], ch, out_sr, RG.tag_field(ref.radio[0])), i
    assert album == RG.analyze_result(hist.astype(np.int32))


def test_long_stream(enc):
    """a C2-length stream (10000 frames of a sweep at 44.1 kHz stereo): many chunks, every window bit-exact"""
    n = 10000 * 1152
    l, r = make_signal("sweep", n, 44100, seed=1)
    got, ref = _check_windows(enc, 2, 44100, 128, l, r)
    assert got["passes"] >= 1


@pytest.mark.parametrize("case", edge_signals.CASES, ids=edge_signals.case_id)
def test_edge_corpus(enc, case):
    kind, ch, sr, kb, frames = case
    if enc.lametag_size(ch, sr, kb) == 0:
        pytest.skip("the tag does not fit: lamejs does not analyse")
    l, r = edge_signals.signal(case)
    _check_windows(enc, ch, sr, kb, l, r)


def test_tag_off_means_no_analysis(enc):
    l, r = make_signal("noise", 20000, 8000, seed=3)
    assert enc.lametag_size(1, 8000, 8) == 0
    streams, title, album = enc.encode_streams_replaygain(1, 8000, 8, [l], None)
    assert title == [RG.GAIN_NOT_ENOUGH_SAMPLES] and album == RG.GAIN_NOT_ENOUGH_SAMPLES
    assert streams == enc.encode_streams_tagged(1, 8000, 8, [l], None)


def test_lametag_build_ex(enc):
    l, r = make_signal("noise", 50000, 44100, seed=4)
    plain = enc.encode_streams_tagged(2, 44100, 128, [l], [r])[0]
    streams, title, _ = enc.encode_streams_replaygain(2, 44100, 128, [l], [r])
    info = enc.get_vbr_tag(plain)
    n = enc.lametag_size(2, 44100, 128)
    crc = oracle_lib.crc16(plain[n:])
    built = enc.lametag_build_ex(2, 44100, 128, info["frames"], len(plain) - n, crc, info["enc_padding"], enc.radio_gain(title[0]))
    assert built == streams[0][:n]
