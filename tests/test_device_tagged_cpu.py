"""The tagged device entry points without a GPU: exported with the arity include/mp3b200.h declares (and the Python binding
passes), and refused with MP3B200_ERR_CUDA when no device is present."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["mp3b200_encode_streams_tagged_device", "mp3b200_encode_streams_tagged_device_f32"]


@pytest.fixture(scope="module")
def M():
    import lamejs_b200

    lamejs_b200.lib()
    return lamejs_b200


def _declared_arity(name):
    hdr = open(os.path.join(ROOT, "include", "mp3b200.h")).read()
    m = re.search(r"\bint\s+%s\s*\(([^)]*)\)\s*;" % name, hdr)
    assert m, name
    return len(m.group(1).split(","))


@pytest.mark.parametrize("name", NAMES)
def test_exported_with_declared_arity(M, name):
    assert _declared_arity(name) == 13
    L = ctypes.CDLL(os.path.join(ROOT, "lamejs_b200", "libmp3b200.so"))
    assert hasattr(L, name)
    assert len(getattr(M.lib(), name).argtypes) == 13


def test_lametag_size_of_resampled_configurations(M):
    """the room a tagged device stream needs: lametag_size(..., resample=True) is mp3b200_lametag_size_ex with
    MP3B200_RESAMPLE (the frame of the rate the configuration encodes at); without the flag such a configuration is refused,
    and a native one answers the same either way (no device needed)"""
    L = M.lib()
    for ch, sr, kb in ((2, 48000, 64), (2, 44100, 48), (1, 32000, 24), (2, 48000, 24)):
        n = M.lametag_size(ch, sr, kb, resample=True)
        assert n == L.mp3b200_lametag_size_ex(ch, sr, kb, M.RESAMPLE) and n >= 0, (ch, sr, kb)
        with pytest.raises(M.Mp3B200Error):
            M.lametag_size(ch, sr, kb)
    assert M.lametag_size(2, 48000, 64, resample=True) == M.lametag_size(2, 24000, 64) > 0
    for ch, sr, kb in ((2, 44100, 128), (1, 8000, 8), (2, 22050, 64)):
        assert M.lametag_size(ch, sr, kb, resample=True) == M.lametag_size(ch, sr, kb) == L.mp3b200_lametag_size(ch, sr, kb)


@pytest.mark.parametrize("name", NAMES)
def test_no_device_is_a_cuda_error(M, name):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    i64 = lambda v: np.array(v, dtype=np.int64)     # noqa: E731
    pcm = np.zeros(4000, dtype=np.float32 if name.endswith("_f32") else np.int16)
    out = np.zeros(8192, dtype=np.uint8)
    pcm_off, ns, out_off, got = i64([0]), i64([4000]), i64([0]), i64([0])
    title = np.zeros(1, dtype=np.float64)
    album = ctypes.c_double(0.0)
    for flags in (0, M.REPLAYGAIN, M.REPLAYGAIN | M.RESAMPLE):
        rc = getattr(M.lib(), name)(1, 44100, 128, flags, 1, pcm.ctypes.data, pcm_off.ctypes.data, ns.ctypes.data, out.ctypes.data,
                                    out_off.ctypes.data, got.ctypes.data, title.ctypes.data, ctypes.byref(album))
        assert rc == -100, flags
    with pytest.raises(M.Mp3B200Error, match="error -100"):
        M.encode_streams_device_tagged(1, 44100, 128, pcm.ctypes.data, [0], [4000], out.ctypes.data, [0],
                                       float32=name.endswith("_f32"), find_replay_gain=True)
