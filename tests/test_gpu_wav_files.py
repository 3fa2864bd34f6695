"""WAV files in, MP3 files out, on the GPU: encode_wav_files against the bytes lamejs made of the hand-made corpus, against
encode_streams / encode_streams_replaygain on rows de-interleaved with numpy, in mixed batches whatever a file's
neighbours are, with ReplayGain across configurations, and k_stage_wav's rows on a poisoned workspace."""
import ctypes
import hashlib
import importlib.util
import json
import os
import random

import numpy as np
import pytest

import lamejs_b200 as M
from synth import make_signal

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "lamejs_wav_golden.json")))
_spec = importlib.util.spec_from_file_location("make_lamejs_wav_golden", os.path.join(HERE, "golden", "make_lamejs_wav_golden.py"))
MAKER = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MAKER)
CORPUS = MAKER.corpus()


def wav_of(ch, sr, frames, seed, kind="noise"):
    """(wav bytes, left, right): a plain 16-bit PCM file of a synth signal and its rows"""
    l, r = make_signal(kind, frames, sr, seed=seed)
    x = np.stack([l, r], axis=1)[:, :ch]
    return MAKER.riff([MAKER.fmt(ch, sr), MAKER.data(np.ascontiguousarray(x, dtype="<i2").tobytes())]), l, r


def test_corpus_equals_lamejs():
    """every file the library encodes gives lamejs's bytes; one call per (kbps, resample), so files share calls"""
    calls = {}
    for name, (wav, kbps, resample) in CORPUS.items():
        calls.setdefault((kbps, resample), []).append(name)
    encoded = 0
    for (kbps, resample), names in calls.items():
        mp3s, status = M.encode_wav_files([CORPUS[n][0] for n in names], kbps, resample=resample)
        for n, mp3, st in zip(names, mp3s, status):
            assert st == M.wav_plan([CORPUS[n][0]], kbps, resample=resample)[0]["status"], n
            if st == M.WAV_ENCODED:
                assert hashlib.sha256(mp3).hexdigest() == GOLD[n]["mp3_sha256"], n
                encoded += 1
            else:
                assert mp3 is None
    assert encoded == sum(1 for n in GOLD if M.wav_plan([CORPUS[n][0]], GOLD[n]["kbps"], resample=GOLD[n]["resample"])[0]["status"] == 0)
    assert encoded >= 14


CASES = [  # (channels, rate, kbps, resample, frames)
    (1, 44100, 128, False, 44100 * 3 + 7),
    (2, 44100, 128, False, 44100 * 3 + 13),
    (1, 22050, 64, False, 30001),
    (2, 16000, 48, False, 20002),
    (1, 8000, 24, False, 9999),
    (2, 24000, 96, False, 25003),
    (2, 48000, 64, True, 48000 + 5),          # lamejs encodes at 24 kHz
    (1, 44100, 32, True, 44100 + 9),          # at 22.05 kHz
    (2, 44100, 48, True, 44100 + 2),          # at 22.05 kHz
]


@pytest.mark.parametrize("ch,sr,kbps,resample,frames", CASES)
def test_equals_encode_streams(ch, sr, kbps, resample, frames):
    files = [wav_of(ch, sr, frames - 1000 * k, 100 + k, kind) for k, kind in enumerate(("noise", "sweep", "burst"))]
    mp3s, status = M.encode_wav_files([f[0] for f in files], kbps, resample=resample)
    assert status == [M.WAV_ENCODED] * 3
    want = M.encode_streams(ch, sr, kbps, [f[1] for f in files], [f[2] for f in files] if ch == 2 else None, resample=resample)
    assert mp3s == want
    tagged, st, title, album = M.encode_wav_files([f[0] for f in files], kbps, resample=resample, find_replay_gain=True)
    w_t, w_title, w_album = M.encode_streams_replaygain(ch, sr, kbps, [f[1] for f in files], [f[2] for f in files] if ch == 2 else None,
                                                        resample=resample)
    assert tagged == w_t and title == w_title and album == w_album
    plain_tag, _ = M.encode_wav_files([f[0] for f in files], kbps, resample=resample, write_vbr_tag=True)
    assert plain_tag == M.encode_streams_tagged(ch, sr, kbps, [f[1] for f in files], [f[2] for f in files] if ch == 2 else None,
                                                resample=resample)


@pytest.mark.parametrize("ch", [1, 2])
def test_sliced_upload(ch):
    """a few long files are uploaded in slices; each slice is staged (stereo) as soon as it lands"""
    files = [wav_of(ch, 44100, 600_001 + 3 * k, 200 + k) for k in range(2)]
    buf = np.zeros(sum(len(f[1]) * ch for f in files), dtype=np.int16)
    arrs = [np.frombuffer(f[0], dtype=np.uint8) for f in files]
    ptrs = (ctypes.c_void_p * 2)(*[a.ctypes.data for a in arrs])
    lens = np.array([len(a) for a in arrs], dtype=np.int64)
    slices = ctypes.c_int32(0)
    assert M.lib().mp3b200_debug_stage_wav(128, 0, 2, ptrs, lens.ctypes.data, buf.ctypes.data, len(buf), ctypes.byref(slices)) == 0
    assert slices.value > 1
    want = np.concatenate([np.concatenate([f[1], f[2]][:ch]) for f in files])
    assert np.array_equal(buf, want)
    mp3s, status = M.encode_wav_files([f[0] for f in files], 128)
    assert mp3s == M.encode_streams(ch, 44100, 128, [f[1] for f in files], [f[2] for f in files] if ch == 2 else None)


def test_stage_wav_writes_every_sample_on_poison():
    """k_stage_wav's rows, on a workspace of 0x7f7f first, equal numpy's de-interleave for every sample: frame counts
    around every multiple of 4 (the kernel's vector width), odd data lengths, one upload slice and many files"""
    rng = np.random.default_rng(7)
    files, want = [], []
    for k, frames in enumerate([0, 1, 2, 3, 4, 5, 7, 8, 9, 1023, 1024, 1025, 4097, 65535, 65538]):
        x = rng.integers(-32768, 32767, size=(frames, 2), dtype=np.int16)
        x[x == 0x7F7F] = 0                                   # the poison never occurs in the input
        extra = b"\x11" * (k % 4)                             # data lengths 4n + 0..3 truncate to n frames
        files.append(MAKER.riff([MAKER.fmt(2, 32000), MAKER.data(x.astype("<i2").tobytes() + extra)]))
        want += [x[:, 0], x[:, 1]]
    want = np.concatenate(want)
    arrs = [np.frombuffer(f, dtype=np.uint8) for f in files]
    ptrs = (ctypes.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
    lens = np.array([len(a) for a in arrs], dtype=np.int64)
    buf = np.zeros(len(want), dtype=np.int16)
    slices = ctypes.c_int32(0)
    assert M.lib().mp3b200_debug_stage_wav(128, 0, len(arrs), ptrs, lens.ctypes.data, buf.ctypes.data, len(buf), ctypes.byref(slices)) == 0
    assert slices.value == 1
    assert not np.any(buf == 0x7F7F)
    assert np.array_equal(buf, want)


def _bad_files():
    """one file of every refused kind"""
    names = ("not_riff", "extended_fmt_40", "stereo_44k_truncated_data", "stereo_44k_streaming_len", "stereo_44k_odd_offset",
             "truncated_header", "mono_44k_8bit", "stereo_44k_float32", "zero_channels")
    bad = [CORPUS[n][0] for n in names]
    bad.append(MAKER.riff([MAKER.fmt(3, 44100), MAKER.data(bytes(600))]))      # three channels: no configuration
    return bad


def test_mixed_batch_in_order_whatever_the_neighbours():
    """three configurations at 64 kbps with resampling (44.1 kHz mono and 22.05 kHz mono native, 48 kHz stereo -> 24 kHz)
    and one file of every refused kind, shuffled"""
    kbps = 64
    good = [(1, 44100, 30000 + 17 * k, 300 + k) for k in range(4)] + [(1, 22050, 15000 + 5 * k, 310 + k) for k in range(3)] + \
           [(2, 48000, 20000 + 3 * k, 320 + k) for k in range(3)]
    good = [(ch, sr) + wav_of(ch, sr, n, seed) for ch, sr, n, seed in good]
    items = [(g[2], i) for i, g in enumerate(good)] + [(b, None) for b in _bad_files()]
    random.Random(5).shuffle(items)
    mp3s, status = M.encode_wav_files([f for f, _ in items], kbps, resample=True)
    assert status == [p["status"] for p in M.wav_plan([f for f, _ in items], kbps, resample=True)]
    assert sum(s == M.WAV_ENCODED for s in status) == len(good)
    assert set(status) == {M.WAV_ENCODED, M.WAV_NOT_WAV, M.WAV_EXTENDED_FMT, M.WAV_RANGE_ERROR, M.WAV_NOT_PCM16, M.WAV_UNSUPPORTED}
    for (f, gi), mp3, st in zip(items, mp3s, status):
        if gi is None:
            assert mp3 is None and st != M.WAV_ENCODED
            continue
        ch, sr, wav, l, r = good[gi]
        assert mp3 == M.encode_streams(ch, sr, kbps, [l], [r] if ch == 2 else None, resample=True)[0]
        assert mp3 == M.encode_wav_files([wav], kbps, resample=True)[0][0]          # alone in a call
    # the good files alone and in another order: the same bytes per file
    order = [i for i, (_, gi) in enumerate(items) if gi is not None][::-1]
    again, st2 = M.encode_wav_files([items[i][0] for i in order], kbps, resample=True)
    assert st2 == [M.WAV_ENCODED] * len(order) and again == [mp3s[i] for i in order]


def test_replaygain_across_configurations():
    groups = {(2, 44100): [wav_of(2, 44100, 44100 + 101 * k, 400 + k, kind) for k, kind in enumerate(("noise", "sweep"))],
              (1, 32000): [wav_of(1, 32000, 32000 + 7 * k, 410 + k, kind) for k, kind in enumerate(("octave", "burst", "noise"))],
              (2, 24000): [wav_of(2, 24000, 24000 + 11 * k, 420 + k) for k in range(2)]}
    kbps = 128
    files, where = [], []
    for key, fs in groups.items():
        for i, f in enumerate(fs):
            files.append(f[0])
            where.append((key, i))
    files.append(_bad_files()[0])
    mp3s, status, title, album = M.encode_wav_files(files, kbps, find_replay_gain=True)
    assert status[-1] == M.WAV_NOT_WAV and mp3s[-1] is None and title[-1] == M.GAIN_NOT_ENOUGH_SAMPLES
    for (ch, sr), fs in groups.items():
        w_mp3, w_title, _ = M.encode_streams_replaygain(ch, sr, kbps, [f[1] for f in fs], [f[2] for f in fs] if ch == 2 else None)
        for (key, i), mp3, t in zip(where, mp3s, title):
            if key == (ch, sr):
                assert mp3 == w_mp3[i] and t == w_title[i]
    encs = []
    for (ch, sr), fs in groups.items():
        for f in fs:
            e = M.Mp3Encoder(ch, sr, kbps, write_vbr_tag=True, find_replay_gain=True)
            e.encodeBuffer(f[1], f[2] if ch == 2 else None)
            e.flush()
            encs.append(e)
    assert album == M.album_gain(encs)
    for e in encs:
        e.close()
