"""SURVEY.md 8(f3), product side, CPU part: the host arithmetic of the tag frame and the WAV reader through the C-ABI (these
entry points need no device), and the decomposition the GPU CRC kernel uses, replayed by g++-compiled k_tag.cuh
(tests/crc_emul.cpp) against the serial CRC of the oracle."""
import ctypes
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import lamejs_b200 as M
from synth import make_signal

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "lamejs_tag_golden.json")))
RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000)
LADDER = [8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160, 192, 224, 256, 320]


@pytest.fixture(scope="module")
def emul():
    d = tempfile.mkdtemp()
    so = os.path.join(d, "crc_emul.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "crc_emul.cpp")])
    E = ctypes.CDLL(so)
    E.emul_range_crc.argtypes = [ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int]
    E.emul_range_crc.restype = ctypes.c_uint
    E.emul_append.argtypes = [ctypes.c_uint, ctypes.c_uint, ctypes.c_ulonglong]
    E.emul_append.restype = ctypes.c_uint
    E.emul_shift.argtypes = [ctypes.c_uint, ctypes.c_ulonglong]
    E.emul_shift.restype = ctypes.c_uint
    return E


def test_crc_kernel_decomposition_equals_serial_crc(oracle, emul):
    """pieces of 512 bytes, 16 bytes per lane, shifts by zero-byte powers, xor in any order == one table look-up per byte"""
    rng = np.random.default_rng(5)
    sizes = list(range(0, 70)) + [511, 512, 513, 1023, 1024, 1025, 4097, 8191, 100003, 417 * 1000 + 333, 4180009]
    for n in sizes:
        a = rng.integers(0, 256, n).astype(np.uint8)
        want = oracle.crc16(a.tobytes())
        for order in (0, 1):
            assert emul.emul_range_crc(a.ctypes.data if n else None, n, order) == want, (n, order)


def test_crc_append_and_shift(oracle, emul):
    rng = np.random.default_rng(6)
    a = rng.integers(0, 256, 6000).astype(np.uint8).tobytes()
    for cut in (0, 1, 417, 418, 5999, 6000):
        assert emul.emul_append(oracle.crc16(a[:cut]), oracle.crc16(a[cut:]), len(a) - cut) == oracle.crc16(a)
    for n in (0, 1, 2, 3, 255, 256, 1000, 123457):
        assert emul.emul_shift(0xBEEF, n) == oracle.crc16(bytes(n), 0xBEEF)
    assert emul.emul_shift(0x1234, (1 << 33) + 5) == emul.emul_shift(emul.emul_shift(0x1234, 1 << 32), (1 << 32) + 5)


def _oracle_tag(oracle, ch, sr, kbps, nframes_hint, seed):
    fs = 1152 if sr >= 32000 else 576
    l, r = make_signal("noise", nframes_hint * fs + seed % 500, sr, seed=seed)
    data, _, info = oracle.encode_stream_tagged(ch, sr, kbps, l, r if ch == 2 else None)
    return info


def test_tag_frame_of_every_configuration_equals_the_oracle(oracle):
    """every (rate, bitrate, channels) the library accepts: size rule of InitVbrTag and all bytes of the frame"""
    n_on = n_off = 0
    for sr in RATES:
        for kbps in LADDER:
            for ch in (1, 2):
                size = M.lib().mp3b200_lametag_size(ch, sr, kbps)
                if oracle.out_samplerate(ch, sr, kbps) != sr:
                    assert size < 0
                    continue
                info = _oracle_tag(oracle, ch, sr, kbps, 3, sr // 100 + kbps + ch)
                if not info["tag_on"]:
                    assert size == 0 and M.lametag_build(ch, sr, kbps, info["frames"] or 5, 1000, 1, 600) == b""
                    n_off += 1
                    continue
                assert size == len(info["tag"])
                got = M.lametag_build(ch, sr, kbps, info["frames"], info["bytes_written"], info["music_crc"], info["encoder_padding"])
                assert got == info["tag"], (ch, sr, kbps)
                n_on += 1
    assert n_on > 200 and n_off > 10


@pytest.mark.parametrize("frames", [1, 2, 99, 100, 101, 399, 400, 401, 799, 800, 801, 1601, 5000])
def test_seek_table_over_frame_counts(oracle, frames):
    """the bag fills to 400 entries, then keeps every second one (VBRTag.js:149-167 with Java's integer index)"""
    ch, sr, kbps = 1, 32000, 32        # 144-byte frames: cheap to encode for real
    l, _ = make_signal("silence", (frames - 2) * 1152 + 600 if frames > 2 else 10, sr, seed=0)
    data, _, info = oracle.encode_stream_tagged(ch, sr, kbps, l, None)
    if sr == 32000 and kbps == 32:
        assert not info["tag_on"]       # 144 < 21 + 156: this configuration carries no tag ...
    ch, sr, kbps = 1, 32000, 48         # ... the next one does (216 bytes)
    data, _, info = oracle.encode_stream_tagged(ch, sr, kbps, l, None)
    assert info["tag_on"] and abs(info["frames"] - frames) <= 1
    got = M.lametag_build(ch, sr, kbps, info["frames"], info["bytes_written"], info["music_crc"], info["encoder_padding"])
    assert got == info["tag"]


@pytest.mark.parametrize("name", sorted(GOLD["wav"]))
def test_wav_header_matches_lamejs(name):
    c = GOLD["wav"][name]
    b, want = bytes.fromhex(c["hex"]), c["result"]
    if "throws" in want:
        with pytest.raises(IndexError if want["throws"] == "RangeError" else ValueError):
            M.WavHeader.readHeader(b)
    elif "undefined" in want:
        assert M.WavHeader.readHeader(b) is None
    else:
        w = M.WavHeader.readHeader(b)
        assert {"dataOffset": w.dataOffset, "dataLen": w.dataLen, "channels": w.channels, "sampleRate": w.sampleRate} == want


def test_wav_header_random_bytes_agree_with_the_oracle(oracle):
    rng = np.random.default_rng(11)
    base = bytes.fromhex(GOLD["wav"]["two_chunks_before_data"]["hex"])
    for _ in range(2000):
        b = bytearray(base)
        for _ in range(int(rng.integers(1, 4))):
            b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
        b = bytes(b[: int(rng.integers(0, len(b) + 1))]) if rng.integers(0, 4) == 0 else bytes(b)
        try:
            want = oracle.wav_read_header(b)
        except (ValueError, IndexError) as e:
            with pytest.raises(type(e)):
                M.WavHeader.readHeader(b)
            continue
        w = M.WavHeader.readHeader(b)
        assert (w is None) == (want is None)
        if w is not None:
            assert {"dataOffset": w.dataOffset, "dataLen": w.dataLen, "channels": w.channels, "sampleRate": w.sampleRate} == want


def test_get_vbr_tag_reads_back_what_the_writer_wrote(oracle):
    """getVbrTag (VBRTag.js:375-470) on the oracle's frames: every rate class and channel mode"""
    for ch, sr, kbps, frames in [(2, 44100, 128, 30), (1, 44100, 128, 5), (2, 48000, 320, 450), (1, 24000, 64, 12), (2, 22050, 64, 12), (1, 8000, 24, 9), (2, 11025, 32, 9)]:
        info = _oracle_tag(oracle, ch, sr, kbps, frames, 77)
        assert info["tag_on"]
        d = M.get_vbr_tag(info["tag"])
        assert d["flags"] == 15 and d["frames"] == info["frames"] and d["bytes"] == info["bytes_written"] + len(info["tag"])
        assert d["samprate"] == sr and d["h_id"] == (1 if sr >= 32000 else 0) and d["headersize"] == len(info["tag"])
        assert d["vbr_scale"] == 57 and d["enc_delay"] == 576 and d["enc_padding"] == info["encoder_padding"]
        x = {True: {1: 21, 2: 36}, False: {1: 13, 2: 21}}[sr >= 32000][ch]
        assert d["toc"] == info["tag"][x + 16:x + 116]
    plain = oracle.encode_stream(2, 44100, 128, *make_signal("noise", 4000, 44100, seed=1))[0]
    assert M.get_vbr_tag(plain[:417]) is None
    with pytest.raises(IndexError):
        M.get_vbr_tag(info["tag"][:20])


def test_crc16_combine(oracle):
    rng = np.random.default_rng(8)
    a = rng.integers(0, 256, 9000).astype(np.uint8).tobytes()
    for cut in (0, 1, 417, 4180, 8999, 9000):
        assert M.crc16_combine(oracle.crc16(a[:cut]), oracle.crc16(a[cut:]), len(a) - cut) == oracle.crc16(a)
    # three segments, as a segment-sharded stream would be combined on rank 0
    parts = [a[:3000], a[3000:7000], a[7000:]]
    c = 0
    for p in parts:
        c = M.crc16_combine(c, oracle.crc16(p), len(p))
    assert c == oracle.crc16(a)


def test_entry_points_reject_bad_arguments_without_a_device():
    """the host-only entry points of this row validate their inputs and never need CUDA"""
    import ctypes
    L = M.lib()
    L.mp3b200_lametag_build.argtypes = [ctypes.c_int] * 3 + [ctypes.c_int64] * 2 + [ctypes.c_int] * 2 + [ctypes.c_void_p, ctypes.c_int]
    buf = np.zeros(2880, dtype=np.uint8)
    assert L.mp3b200_lametag_size(2, 44100, 64) < 0 and L.mp3b200_lametag_size(3, 44100, 128) < 0      # lamejs would resample / bad channels
    assert L.mp3b200_lametag_build(2, 44100, 64, 10, 1000, 0, 576, buf.ctypes.data, 2880) < 0
    assert L.mp3b200_lametag_build(2, 44100, 128, 0, 0, 0, 576, buf.ctypes.data, 2880) == 0            # no frame counted: no tag
    assert L.mp3b200_lametag_build(2, 44100, 128, 10, 4170, 0, 576, None, 0) == 417                    # size query
    assert L.mp3b200_lametag_build(2, 44100, 128, 10, 4170, 0, 576, buf.ctypes.data, 100) == 417 and not buf.any()
    assert L.mp3b200_wav_read_header(None, 0, None) < 0 and L.mp3b200_get_vbr_tag(None, 10, None) < 0
    L.mp3b200_crc16_combine.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int64]
    assert L.mp3b200_crc16_combine(1, 2, -1) < 0 and L.mp3b200_crc16_combine(0x1234, 0, 0) == 0x1234
    # handle entry points with a NULL handle
    L.mp3b200_put_vbr_tag.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
    assert L.mp3b200_set_write_vbr_tag(None, 1) == -3 and L.mp3b200_get_lametag_frame(None, None, 0) == -3 and L.mp3b200_put_vbr_tag(None, None, 0) == -3
    assert L.mp3b200_music_crc(None) == -1 and L.mp3b200_bytes_written(None) == -1


@pytest.mark.parametrize("ch,sr,kbps", [(2, 44100, 130), (2, 44100, 120), (1, 44100, 100), (2, 48000, 300), (1, 32000, 70), (2, 24000, 50), (1, 16000, 60), (2, 48000, 1000),
                                        (1, 44100, 72), (1, 32000, 52), (2, 12000, 36), (2, 8000, 28), (2, 44100, 104)])
def test_tag_frame_with_bitrates_off_the_ladder(oracle, ch, sr, kbps):
    """kbps is snapped like FindNearestBitrate, but the low-pass (a tag field) comes from the rate as given (Lame.js:838-885 runs
    before :1053): the tag must follow both"""
    if oracle.out_samplerate(ch, sr, kbps) != sr:
        assert M.lib().mp3b200_lametag_size(ch, sr, kbps) < 0
        return
    info = _oracle_tag(oracle, ch, sr, kbps, 4, 5)
    size = M.lib().mp3b200_lametag_size(ch, sr, kbps)
    if not info["tag_on"]:
        assert size == 0
        return
    assert size == len(info["tag"])
    assert M.lametag_build(ch, sr, kbps, info["frames"], info["bytes_written"], info["music_crc"], info["encoder_padding"]) == info["tag"]
