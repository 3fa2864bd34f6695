"""Encode sessions without a GPU: the entry points are exported with the arity include/mp3b200.h declares (and the Python
binding passes), a session cannot be created without a device, and mp3b200_check_status maps the status words to the
synchronous call's errors on the host."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARITY = {"mp3b200_session_create": 2, "mp3b200_session_destroy": 1, "mp3b200_encode_streams_async": 12,
         "mp3b200_encode_streams_async_f32": 12, "mp3b200_check_status": 1}


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


def test_no_device_is_a_cuda_error(M):
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = ctypes.c_void_p()
    assert M.lib().mp3b200_session_create(None, ctypes.byref(h)) == -100
    assert b"no CUDA device" in M.lib().mp3b200_last_error()
    assert not h.value


def test_null_arguments_are_handle_errors(M):
    L = M.lib()
    assert L.mp3b200_session_create(None, None) == -3
    assert L.mp3b200_session_destroy(None) == -3
    assert L.mp3b200_encode_streams_async(None, 2, 44100, 128, 0, 1, None, None, None, None, None, None) == -3
    assert L.mp3b200_encode_streams_async_f32(None, 2, 44100, 128, 0, 1, None, None, None, None, None, None) == -3
    assert L.mp3b200_check_status(None) == -3


@pytest.mark.parametrize("words,rc,text", [
    ([0, 0, 2, 0], 0, None),
    ([0, 0, 7, 0], 0, None),
    ([1, 0, 2, 0], -1, b"non-finite input sample (or one beyond 2^40 once scaled)"),
    ([0, 3, 2, 0], -1, b"frame over its bit budget (input too loud to encode)"),
    ([1, 3, 2, 0], -1, b"non-finite input sample (or one beyond 2^40 once scaled)"),
    ([0, 0, 99, 1], -100, b"quantizer stage failed: the fixed-point loop did not converge"),
])
def test_check_status(M, words, rc, text):
    w = np.array(words, dtype=np.int32)
    assert M.lib().mp3b200_check_status(w.ctypes.data) == rc
    if text is not None:
        assert M.lib().mp3b200_last_error() == text
