"""The streaming calls fed from device memory without a GPU: exported with the arity include/mp3b200.h declares (and the
Python binding passes), and refused with MP3B200_ERR_CUDA when no device is present."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARITY = {"mp3b200_encode_device": 6, "mp3b200_encode_device_f32": 6, "mp3b200_encode_batch_device": 8,
         "mp3b200_encode_batch_device_f32": 8}


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


@pytest.mark.parametrize("name", sorted(ARITY))
def test_exported_with_declared_arity(M, name):
    assert _declared_arity(name) == ARITY[name]
    L = ctypes.CDLL(os.path.join(ROOT, "lamejs_b200", "libmp3b200.so"))
    assert hasattr(L, name)
    assert len(getattr(M.lib(), name).argtypes) == ARITY[name]


@pytest.mark.parametrize("name", sorted(ARITY))
def test_no_device_is_a_cuda_error(M, name):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    pcm = np.zeros(4000, dtype=np.float32 if name.endswith("_f32") else np.int16)
    out = np.zeros(8192, dtype=np.uint8)
    fn = getattr(M.lib(), name)
    if "batch" in name:
        vp = ctypes.c_void_p
        hs, rows, op = (vp * 1)(None), (vp * 1)(pcm.ctypes.data), (vp * 1)(out.ctypes.data)
        ns, cap, got = np.array([4000], np.int32), np.array([8192], np.int32), np.zeros(1, np.int32)
        rc = fn(hs, rows, None, ns.ctypes.data, op, cap.ctypes.data, 1, got.ctypes.data)
    else:
        rc = fn(None, pcm.ctypes.data, None, 4000, out.ctypes.data, 8192)
    assert rc == -100
    assert b"no CUDA device" in M.lib().mp3b200_last_error()
