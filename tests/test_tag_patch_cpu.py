"""The bytes of a tag frame that depend on the encoded data -- music CRC, Radio Replay Gain field, the tag's own CRC -- are
written by one set of __host__ __device__ functions (lamejs_b200/csrc/k_tag.cuh): mp3_tag_frame ends in them and k_tag_finish
completes a host-built template with them on the device.  tests/tag_patch_emul.cpp compiles them with g++; a template frame
patched there must equal the frame the library builds directly from the same numbers, for every configuration."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

import lamejs_b200 as M

HERE = os.path.dirname(os.path.abspath(__file__))
RATES = (8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000)
LADDER = [8, 16, 24, 32, 40, 48, 56, 64, 80, 96, 112, 128, 144, 160, 192, 224, 256, 320]
GAINS = [M.GAIN_NOT_ENOUGH_SAMPLES, -51.1, -51.0, -50.95, -0.05, -0.04, 0.0, 0.04, 0.05, -7.36, 3.21, 50.95, 51.0, 51.1, 64.82]


@pytest.fixture(scope="module")
def emul():
    d = tempfile.mkdtemp()
    so = os.path.join(d, "tag_patch_emul.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "tag_patch_emul.cpp")])
    E = ctypes.CDLL(so)
    E.emul_radio_gain.argtypes = [ctypes.c_double]
    E.emul_patch.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_double]
    E.emul_patch.restype = None
    return E


def _configs():
    """(ch, sr, kbps, resample) of every configuration that carries a tag, native and resampled"""
    for sr in RATES:
        for kbps in LADDER:
            for ch in (1, 2):
                native = M.out_samplerate(ch, sr, kbps) == sr
                if M.lib().mp3b200_lametag_size_ex(ch, sr, kbps, 0 if native else M.RESAMPLE) > 0:
                    yield ch, sr, kbps, not native


def _sideinfo_len(ch, out_sr):
    return 4 + ((32 if ch == 2 else 17) if out_sr >= 32000 else (17 if ch == 2 else 9))


def test_radio_gain_and_field(emul):
    rng = np.random.default_rng(21)
    for db in GAINS + list(rng.uniform(-70, 70, 500)) + [k / 20 for k in range(-1100, 1100)]:
        rg = emul.emul_radio_gain(db)
        assert rg == M.radio_gain(db), db
        mag = min(abs(rg), 0x1FE)
        assert emul.emul_radio_gain_field(rg) == 0x2C00 | (0x200 if rg < 0 else 0) | mag, db
    assert emul.emul_radio_gain_field(emul.emul_radio_gain(M.GAIN_NOT_ENOUGH_SAMPLES)) == 0x2C00 | 0x200 | 0x1FE


def test_patched_template_equals_the_frame_built_directly(emul):
    rng = np.random.default_rng(22)
    n = 0
    for ch, sr, kbps, rs in _configs():
        side = _sideinfo_len(ch, M.out_samplerate(ch, sr, kbps))
        assert emul.emul_head_bytes(side) <= M.lametag_size(ch, sr, kbps, resample=rs)
        for k in range(4):
            frames = int(rng.choice([1, 2, 99, 401, 10001])) if k == 0 else int(rng.integers(1, 30000))
            music = int(rng.integers(1, 1 << 28))
            padding = int(rng.integers(576, 2881))
            crc = int(rng.integers(0, 1 << 16)) if k else 0xFFFF
            db = GAINS[(n + k) % len(GAINS)] if k < 3 else float(rng.uniform(-60, 60))
            want = M.lametag_build_ex(ch, sr, kbps, frames, music, crc, padding, M.radio_gain(db), resample=rs)
            # a frame of the same stream with other data-dependent bytes: the patch must overwrite all of them
            other = M.lametag_build_ex(ch, sr, kbps, frames, music, crc ^ 0x5A5A, padding, M.radio_gain(db) + 7, resample=rs)
            assert other != want
            buf = np.frombuffer(other, dtype=np.uint8).copy()
            emul.emul_patch(buf.ctypes.data, side, crc, 1, db)
            assert buf.tobytes() == want, (ch, sr, kbps, frames, crc, db)
            if not rs:
                # the template the session uploads (music CRC 0, field 0), and a stream nobody analysed
                tpl = np.frombuffer(M.lametag_build(ch, sr, kbps, frames, music, 0, padding), dtype=np.uint8).copy()
                emul.emul_patch(tpl.ctypes.data, side, crc, 1, db)
                assert tpl.tobytes() == want
                emul.emul_patch(tpl.ctypes.data, side, crc, 0, 0.0)
                assert tpl.tobytes() == M.lametag_build(ch, sr, kbps, frames, music, crc, padding)
            n += 1
    assert n > 250
