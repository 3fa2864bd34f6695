"""WAV files in, MP3 files out, host side (no device): mp3b200_wav_plan against what lamejs made of the hand-made corpus
(tests/golden/lamejs_wav_golden.json), a fuzz of header bytes against the oracle's readHeader plus the Int16Array view
rule, and the argument gate of mp3b200_encode_wav / _tagged, which answers before any CUDA call."""
import ctypes
import hashlib
import importlib.util
import json
import os
import struct

import numpy as np
import pytest

import lamejs_b200 as M
from lamejs_b200.encoder import WAV_TAG

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "lamejs_wav_golden.json")))
_spec = importlib.util.spec_from_file_location("make_lamejs_wav_golden", os.path.join(HERE, "golden", "make_lamejs_wav_golden.py"))
MAKER = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MAKER)
CORPUS = MAKER.corpus()


def _fmt_fields(wav):
    """the fmt chunk's format tag and bits per sample (readHeader never reads them)"""
    return struct.unpack_from("<H", wav, 20)[0], struct.unpack_from("<H", wav, 34)[0]


def test_corpus_is_the_one_lamejs_ran():
    assert sorted(CORPUS) == sorted(GOLD)
    for name, (wav, kbps, resample) in CORPUS.items():
        assert hashlib.sha256(wav).hexdigest() == GOLD[name]["wav_sha256"], name
        assert (kbps, resample) == (GOLD[name]["kbps"], GOLD[name]["resample"])


@pytest.mark.parametrize("name", sorted(GOLD))
def test_plan_gives_lamejs_outcome(name):
    wav, kbps, resample = CORPUS[name]
    g = GOLD[name]
    p = M.wav_plan([wav], kbps, resample=resample)[0]
    pt = M.wav_plan([wav], kbps, resample=resample, write_vbr_tag=True)[0]
    assert {k: v for k, v in p.items() if k != "out_bytes"} == {k: v for k, v in pt.items() if k != "out_bytes"}
    if g.get("undefined"):
        assert p["status"] == M.WAV_NOT_WAV
        return
    if g.get("throws") == "extended fmt chunk not implemented":
        assert p["status"] == M.WAV_EXTENDED_FMT
        return
    if g.get("throws") == "RangeError":
        assert p["status"] == M.WAV_RANGE_ERROR
        assert p["nsamples"] == 0 and p["out_bytes"] == 0
        return
    assert "mp3_sha256" in g, g                   # lamejs encoded it
    h = g["header"]
    assert (p["channels"], p["sample_rate"], p["data_offset"]) == (h["channels"], h["sampleRate"], h["dataOffset"])
    assert p["nsamples"] == g["left_len"]
    if g["right_len"] >= 0:
        assert g["right_len"] == g["left_len"]
    if _fmt_fields(wav) != (1, 16):               # the deviation: lamejs encoded Int16 noise, the library refuses
        assert p["status"] == M.WAV_NOT_PCM16 and p["out_bytes"] == 0
        return
    flags = M.RESAMPLE if resample else 0
    if M.lib().mp3b200_stream_bytes_ex(h["channels"], h["sampleRate"], kbps, flags, 0) < 0:
        assert p["status"] == M.WAV_UNSUPPORTED and p["out_bytes"] == 0
        return
    assert p["status"] == M.WAV_ENCODED
    assert p["out_samplerate"] == M.out_samplerate(h["channels"], h["sampleRate"], kbps)
    nb = M.lib().mp3b200_stream_bytes_ex(h["channels"], h["sampleRate"], kbps, flags, g["left_len"])
    assert p["out_bytes"] == nb == g["mp3_bytes"]
    assert pt["out_bytes"] == nb + M.lib().mp3b200_lametag_size_ex(h["channels"], h["sampleRate"], kbps, flags)


def test_corpus_covers_every_status():
    seen = {M.wav_plan([w], k, resample=r)[0]["status"] for w, k, r in CORPUS.values()}
    assert seen == {M.WAV_ENCODED, M.WAV_NOT_WAV, M.WAV_EXTENDED_FMT, M.WAV_RANGE_ERROR, M.WAV_NOT_PCM16, M.WAV_UNSUPPORTED}


def _expected(oracle, wav, kbps, resample):
    """status and samples per channel from the oracle's readHeader, the Int16Array rules and the configuration rule"""
    try:
        h = oracle.wav_read_header(wav)
    except ValueError:
        return M.WAV_EXTENDED_FMT, 0
    except IndexError:
        return M.WAV_RANGE_ERROR, 0
    if h is None:
        return M.WAV_NOT_WAV, 0
    off, dl, ch, sr = h["dataOffset"], h["dataLen"], h["channels"], h["sampleRate"]
    view = dl // 2
    if off % 2 or off + 2 * view > len(wav) or (ch == 0 and dl > 0):
        return M.WAV_RANGE_ERROR, 0
    n = view if ch == 1 else (0 if ch == 0 else dl // (2 * ch))
    if _fmt_fields(wav) != (1, 16):
        return M.WAV_NOT_PCM16, n
    if sr >= 2 ** 31 or M.lib().mp3b200_stream_bytes_ex(ch, sr, kbps, M.RESAMPLE if resample else 0, 0) < 0:
        return M.WAV_UNSUPPORTED, n
    return M.WAV_ENCODED, n


def test_fuzzed_headers_agree_with_oracle(oracle):
    rng = np.random.default_rng(20261019)
    seeds = [w for w, _, _ in CORPUS.values() if len(w) >= 44]
    kbps_ladder = [8, 32, 64, 96, 128, 192, 320]
    for it in range(3000):
        wav = bytearray(seeds[rng.integers(len(seeds))][:600])
        op = rng.integers(6)
        if op == 0:                                           # random bytes anywhere in the first 64
            for _ in range(rng.integers(1, 4)):
                wav[rng.integers(min(64, len(wav)))] = rng.integers(256)
        elif op == 1:                                         # a random cut
            wav = wav[: rng.integers(len(wav) + 1)]
        elif op == 2:                                         # a random data length
            at = wav.find(b"data")
            if at >= 0:
                wav[at + 4: at + 8] = struct.pack("<I", int(rng.choice([0, 1, 2, 3, 5, 0xFFFFFFFF, rng.integers(1 << 32)])))
        elif op == 3:                                         # channels / rate / tag / bits
            field = [(22, "<H", [0, 1, 2, 3, 6, 65535]), (24, "<I", [8000, 11025, 44100, 48000, 96000, 0, 0xFFFFFFFF]),
                     (20, "<H", [1, 3, 0xFFFE]), (34, "<H", [8, 16, 24, 32])][rng.integers(4)]
            struct.pack_into(field[1], wav, field[0], int(rng.choice(field[2])))
        elif op == 4:                                         # fmt length
            struct.pack_into("<I", wav, 16, int(rng.choice([14, 16, 17, 18, 20, 40])))
        else:                                                 # a chunk of random length before the data
            chunk = b"junk" + struct.pack("<I", int(rng.integers(0, 9))) + bytes(int(rng.integers(0, 9)))
            wav = wav[:36] + chunk + wav[36:]
        kbps, resample = int(rng.choice(kbps_ladder)), bool(rng.integers(2))
        p = M.wav_plan([bytes(wav)], kbps, resample=resample)[0]
        want = _expected(oracle, bytes(wav), kbps, resample)
        assert (p["status"], p["nsamples"]) == want, (it, bytes(wav[:48]).hex(), kbps, resample, p)


def _call(L, fn, kbps, flags, files, nfiles=None, lens=None, out=True, cap=None, status=True, title=None):
    n = len(files) if nfiles is None else nfiles
    arrs = [np.frombuffer(f, dtype=np.uint8) if f is not None else None for f in files]
    ptrs = (ctypes.c_void_p * max(len(files), 1))(*[None if a is None else a.ctypes.data for a in arrs])
    lens = np.array([len(f) if f is not None else 0 for f in files] if lens is None else lens, dtype=np.int64)
    bufs = [np.zeros(8192, dtype=np.uint8) for _ in files]
    op = (ctypes.c_void_p * max(len(files), 1))(*[b.ctypes.data for b in bufs])
    caps = np.array([8192] * len(files) if cap is None else cap, dtype=np.int64)
    got = np.full(max(len(files), 1), -7, dtype=np.int64)
    st = np.full(max(len(files), 1), -7, dtype=np.int32)
    args = [kbps, flags, n, ptrs, lens.ctypes.data, op if out else None, caps.ctypes.data, got.ctypes.data, st.ctypes.data if status else None]
    if fn == "tagged":
        t = np.zeros(max(len(files), 1))
        a = ctypes.c_double(0)
        rc = L.mp3b200_encode_wav_tagged(*args, t.ctypes.data, ctypes.byref(a))
        return rc, got, st, t, a.value
    return L.mp3b200_encode_wav(*args), got, st


def test_argument_gate_without_a_device():
    """every refusal comes before any CUDA call, so it is the same here as on a GPU; files that are all refused need no
    device either, and get their statuses"""
    L = M.lib()
    good = CORPUS["stereo_44k"][0]
    E_H, E_C, E_B = -3, -1, -1
    assert _call(L, "plain", 128, 0, [good], nfiles=-1)[0] == E_H
    assert _call(L, "plain", 128, M.REPLAYGAIN, [good])[0] == E_C          # the tagged call's flag
    assert _call(L, "plain", 128, WAV_TAG, [good])[0] == E_C                  # the plan's flag
    assert _call(L, "tagged", 128, 8, [good])[0] == E_C
    assert _call(L, "plain", 128, 0, [good], out=False)[0] == E_H
    assert _call(L, "plain", 128, 0, [good], status=False)[0] == E_H
    assert _call(L, "plain", 128, 0, [None])[0] == E_H                     # NULL file
    assert _call(L, "plain", 128, 0, [good], lens=[-1])[0] == E_H
    assert _call(L, "plain", 128, 0, [good], cap=[100])[0] == E_B          # too small for a file that is encoded
    assert L.mp3b200_encode_wav(128, 0, 1, None, None, None, None, None, None) == E_H
    assert L.mp3b200_encode_wav(128, 0, 0, None, None, None, None, None, None) == 0
    # with ReplayGain, more than 65535 files are refused before anything is read
    many = [b"x"] * 65536
    assert _call(L, "tagged", 128, M.REPLAYGAIN, many)[0] == E_H
    # the plan: its own flags, a NULL plan
    assert L.mp3b200_wav_plan(128, M.REPLAYGAIN, 0, None, None, None) == E_C
    assert L.mp3b200_wav_plan(128, 0, 1, None, None, None) == E_H
    # only refused files: statuses, nothing encoded, no device touched; a tiny cap does not matter for them
    bad = [CORPUS[k][0] for k in ("not_riff", "extended_fmt_40", "truncated_header", "mono_44k_8bit", "mono_44k_8kbps", "zero_channels")]
    rc, got, st = _call(L, "plain", 8, 0, bad, cap=[0] * len(bad))
    assert rc == 0 and list(got) == [0] * len(bad)
    assert list(st) == [M.WAV_NOT_WAV, M.WAV_EXTENDED_FMT, M.WAV_RANGE_ERROR, M.WAV_NOT_PCM16, M.WAV_UNSUPPORTED, M.WAV_RANGE_ERROR]
    rc, got, st, title, album = _call(L, "tagged", 8, M.REPLAYGAIN, bad)
    assert rc == 0 and list(title[:len(bad)]) == [M.GAIN_NOT_ENOUGH_SAMPLES] * len(bad) and album == M.GAIN_NOT_ENOUGH_SAMPLES
    rc, got, st, title, album = _call(L, "tagged", 8, M.REPLAYGAIN, [])
    assert rc == 0 and album == M.GAIN_NOT_ENOUGH_SAMPLES
